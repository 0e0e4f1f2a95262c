"""Random affine augmentation of a batch, every image with its own parameters: torchvision's ``transforms.v2.RandomAffine``
definition, drawn and applied on the device in one launch (``ops.random_affine``), so that it can run inside a captured training
step (``engine.GraphedTrainStep(augment=...)``)."""
from __future__ import annotations

import math
import numbers
from collections.abc import Sequence
from typing import Optional

import torch


def _check_sequence_input(x, name, req_sizes):
    msg = req_sizes[0] if len(req_sizes) < 2 else " or ".join([str(s) for s in req_sizes])
    if not isinstance(x, Sequence):
        raise TypeError(f"{name} should be a sequence of length {msg}.")
    if len(x) not in req_sizes:
        raise ValueError(f"{name} should be a sequence of length {msg}.")


def _setup_angle(x, name, req_sizes=(2,)):
    if isinstance(x, numbers.Number):
        if x < 0:
            raise ValueError(f"If {name} is a single number, it must be positive.")
        x = [-x, x]
    else:
        _check_sequence_input(x, name, req_sizes)
    return [float(d) for d in x]


class RandomAffine:
    """Random rotation, translation, scaling and shear of every image of an fp32 ``[B, C, H, W]`` batch about its centre, each image
    with its own parameters.  The arguments, their checks and their error messages are torchvision's ``RandomAffine`` (without
    ``center``; ``fill`` is one number).  Per image, with torchvision's ``make_params``:

        angle ~ U[degrees),  tx = round(U[-translate[0]·W, translate[0]·W))  (ty likewise with H; 0 without translate),
        scale ~ U[scale) (1 without),  shear_x ~ U[shear[0], shear[1]),  shear_y ~ U[shear[2], shear[3]) with four values (else 0)

    drawn in fp32 and rounded half to even; the image is then resampled as torchvision's ``affine`` does (``interpolation``
    ``"nearest"`` or ``"bilinear"``, ``fill`` where the source lies outside the image).

    * A CUDA batch takes the native kernel: one launch, parameters drawn on the device from ``generator`` (a CUDA generator on the
      batch's device; the default one when None), nothing on the host, capturable in a CUDA graph where every replay draws new
      parameters.  ``torch.manual_seed`` (or the generator's ``manual_seed``) reproduces the sequence.
    * A CPU batch takes torch ops with the same definition, drawing from ``generator`` (a CPU generator; torch's default one when
      None).
    * Any other dtype raises ``TypeError``.

    ``record_params=True`` keeps the last call's parameters in ``last_params``: fp32 ``[B, 6]`` (angle, tx, ty, scale, shear_x,
    shear_y) on the batch's device.  Inside a CUDA graph it is the graph's static tensor, holding the last replay's draws."""

    def __init__(self, degrees, translate=None, scale=None, shear=None, interpolation="nearest", fill: float = 0.0,
                 generator: Optional[torch.Generator] = None, record_params: bool = False):
        self.degrees = _setup_angle(degrees, name="degrees", req_sizes=(2,))
        if translate is not None:
            _check_sequence_input(translate, "translate", req_sizes=(2,))
            for t in translate:
                if not (0.0 <= t <= 1.0):
                    raise ValueError("translation values should be between 0 and 1")
            translate = [float(t) for t in translate]
        self.translate = translate
        if scale is not None:
            _check_sequence_input(scale, "scale", req_sizes=(2,))
            for s in scale:
                if s <= 0:
                    raise ValueError("scale values should be positive")
            scale = [float(s) for s in scale]
        self.scale = scale
        self.shear = None if shear is None else _setup_angle(shear, name="shear", req_sizes=(2, 4))
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

    def __repr__(self) -> str:
        return (f"RandomAffine(degrees={self.degrees}, translate={self.translate}, scale={self.scale}, shear={self.shear}, "
                f"interpolation={self.interpolation!r}, fill={self.fill})")

    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        if images.dtype != torch.float32:
            raise TypeError(f"RandomAffine: images must be float32 (got {images.dtype})")
        if images.dim() != 4:
            raise ValueError(f"RandomAffine: images must be [B, C, H, W] (got shape {tuple(images.shape)})")
        if images.is_cuda:
            from .. import ops

            out, params = ops.random_affine(images.contiguous(), self.degrees, self.translate, self.scale, self.shear,
                                            bilinear=self.interpolation == "bilinear", fill=self.fill, generator=self.generator,
                                            record_params=self.record_params)
        else:
            out, params = _random_affine_cpu(images, self.degrees, self.translate, self.scale, self.shear,
                                             self.interpolation == "bilinear", self.fill, self.generator)
        if self.record_params:
            self.last_params = params
        return out


def _random_affine_cpu(x, degrees, translate, scale, shear, bilinear, fill, generator):
    """The CPU path of RandomAffine: the kernel's definition in torch ops, coordinates and weights in float64."""
    B, C, H, W = x.shape

    def draw(lo, hi):
        return torch.empty(B).uniform_(lo, hi, generator=generator)

    zeros = torch.zeros(B)
    angle = draw(*degrees)
    if translate is not None:
        max_dx, max_dy = float(translate[0] * W), float(translate[1] * H)
        tx, ty = torch.round(draw(-max_dx, max_dx)), torch.round(draw(-max_dy, max_dy))   # half to even
    else:
        tx, ty = zeros, zeros
    sc = draw(*scale) if scale is not None else torch.ones(B)
    shx = draw(shear[0], shear[1]) if shear is not None else zeros
    shy = draw(shear[2], shear[3]) if shear is not None and len(shear) == 4 else zeros
    params = torch.stack([angle, tx, ty, sc, shx, shy], 1)
    if B == 0:
        return x.clone(), params
    # torchvision's _get_inverse_affine_matrix with center (0, 0), in float64
    p = params.double()
    rad = math.pi / 180.0
    rot, sx, sy = p[:, 0] * rad, p[:, 4] * rad, p[:, 5] * rad
    a = torch.cos(rot - sy) / torch.cos(sy)
    b = -torch.cos(rot - sy) * torch.tan(sx) / torch.cos(sy) - torch.sin(rot)
    c = torch.sin(rot - sy) / torch.cos(sy)
    d = -torch.sin(rot - sy) * torch.tan(sx) / torch.cos(sy) + torch.cos(rot)
    s = p[:, 3]
    m0, m1, m3, m4 = d / s, -b / s, -c / s, a / s
    m2 = m0 * -p[:, 1] + m1 * -p[:, 2]
    m5 = m3 * -p[:, 1] + m4 * -p[:, 2]
    cw, ch = 0.5 * (W - 1), 0.5 * (H - 1)
    xj = (torch.arange(W, dtype=torch.float64) - cw).view(1, 1, W)
    yi = (torch.arange(H, dtype=torch.float64) - ch).view(1, H, 1)
    col = lambda v: v.view(B, 1, 1)   # noqa: E731
    src_x = col(m0) * xj + col(m1) * yi + col(m2) + cw
    src_y = col(m3) * xj + col(m4) * yi + col(m5) + ch
    return _sample_cpu(x, src_x, src_y, bilinear, fill), params


def _sample_cpu(x, src_x, src_y, bilinear, fill):
    """Every channel of x [B, C, H, W] sampled at the float64 source coordinates src_x, src_y [B, H, W]: grid_sample
    (align_corners=False, padding_mode="zeros") unnormalised; nearest rounds half to even and takes ``fill`` outside the image,
    bilinear (in float64) returns torchvision's (v − fill)·mask + fill."""
    B, C, H, W = x.shape
    flat = x.reshape(B, C, H * W)

    def tap(ix, iy):
        """(in bounds, value) of the integer-valued coordinates ix, iy [B, H, W]; 0 outside"""
        inside = (ix >= 0) & (ix <= W - 1) & (iy >= 0) & (iy <= H - 1)
        idx = torch.where(inside, iy * W + ix, 0).long().view(B, 1, H * W).expand(B, C, H * W)
        v = torch.gather(flat, 2, idx).view(B, C, H, W)
        return inside, torch.where(inside.unsqueeze(1), v, 0)

    if not bilinear:
        inside, v = tap(torch.round(src_x), torch.round(src_y))
        return torch.where(inside.unsqueeze(1), v, torch.tensor(fill, dtype=x.dtype))
    x0, y0 = torch.floor(src_x), torch.floor(src_y)
    fx, fy = src_x - x0, src_y - y0
    acc = torch.zeros(B, C, H, W, dtype=torch.float64)
    mask = torch.zeros(B, H, W, dtype=torch.float64)
    for dx, dy, w in ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy)):
        inside, v = tap(x0 + dx, y0 + dy)
        w = torch.where(inside, w, 0)
        acc += w.unsqueeze(1) * v.double()
        mask += w
    return ((acc - fill) * mask.unsqueeze(1) + fill).to(x.dtype)
