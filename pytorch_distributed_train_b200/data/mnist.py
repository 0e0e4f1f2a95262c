"""MNIST dataset without PIL or the network.

The reference builds ``torchvision.datasets.MNIST(root='./data', train=True,
transform=ToTensor(), download=True)`` (ref: ddp_example.py:66-69), which downloads four
idx-ubyte archives and converts every sample through PIL on the training thread.  Here:

* the idx files are parsed directly (``root/MNIST/raw/*-ubyte[.gz]``, the layout torchvision
  writes, so an existing download is picked up as is);
* samples stay a uint8 tensor; ``__getitem__`` yields what ``ToTensor`` would
  (float32 ``[1,28,28]`` in ``[0,1]``, int label) and ``gather(indices)`` builds a whole batch
  with one ``index_select`` + one cast;
* ``download=True`` fetches the four archives from the mirrors torchvision uses and verifies their md5 sums
  (tv datasets/mnist.py:37-47,174-197) — when a network is reachable.  The GPU boxes of this project have none, so a
  short connectivity probe decides: unreachable + ``synthetic_fallback=True`` writes deterministic synthetic idx files
  of the real shape (60000/10000 × 28×28) so the full file-parsing path still runs; unreachable without the fallback
  raises with instructions.
"""
from __future__ import annotations

import gzip
import os
import struct
from typing import Callable, Optional, Sequence, Tuple

import torch

_FILES = {
    True: ("train-images-idx3-ubyte", "train-labels-idx1-ubyte", 60000),
    False: ("t10k-images-idx3-ubyte", "t10k-labels-idx1-ubyte", 10000),
}


# mirrors and checksums of the reference's dataset (torchvision.datasets.MNIST)
_MIRRORS = ("https://ossci-datasets.s3.amazonaws.com/mnist/", "http://yann.lecun.com/exdb/mnist/")
_MD5 = {
    "train-images-idx3-ubyte.gz": "f68b3c2dcbeaaa9fbdd348bbdeb94873",
    "train-labels-idx1-ubyte.gz": "d53e105ee54ea40749a09fcbcd1e9432",
    "t10k-images-idx3-ubyte.gz": "9fb629c4189551a2d022fa330f9573f3",
    "t10k-labels-idx1-ubyte.gz": "ec29112dd5afa0611ce80d1b7f02629c",
}


def _md5(path: str) -> str:
    import hashlib

    h = hashlib.md5()
    with open(path, "rb") as f:
        for chunk in iter(lambda: f.read(1 << 20), b""):
            h.update(chunk)
    return h.hexdigest()


def network_reachable(timeout: float = 2.0) -> bool:
    """Cheap probe (one TCP connect) so an offline box fails in seconds, not after urllib's retries."""
    import socket

    for host, port in (("ossci-datasets.s3.amazonaws.com", 443), ("yann.lecun.com", 80)):
        try:
            with socket.create_connection((host, port), timeout=timeout):
                return True
        except OSError:
            continue
    return False


def download_mnist(root: str, timeout: float = 30.0) -> bool:
    """Fetch + verify the four MNIST archives into ``root/MNIST/raw`` (ref: ddp_example.py:66-69 ``download=True``).
    Returns False when no network is reachable; raises if a download is corrupt."""
    import urllib.request

    raw = os.path.join(root, "MNIST", "raw")
    missing = [n for n in _MD5 if not (os.path.exists(os.path.join(raw, n)) and _md5(os.path.join(raw, n)) == _MD5[n])
               and not os.path.exists(os.path.join(raw, n[:-3]))]
    if not missing:
        return True
    if not network_reachable():
        return False
    os.makedirs(raw, exist_ok=True)
    for name in missing:
        dst, err = os.path.join(raw, name), None
        for mirror in _MIRRORS:
            try:
                tmp = dst + f".part{os.getpid()}"
                with urllib.request.urlopen(mirror + name, timeout=timeout) as r, open(tmp, "wb") as f:
                    while True:
                        chunk = r.read(1 << 16)
                        if not chunk:
                            break
                        f.write(chunk)
                if _md5(tmp) != _MD5[name]:
                    os.remove(tmp)
                    raise RuntimeError(f"md5 mismatch for {name} from {mirror}")
                os.replace(tmp, dst)
                err = None
                break
            except Exception as e:  # noqa: BLE001 - try the next mirror
                err = e
        if err is not None:
            raise RuntimeError(f"MNIST download failed for {name}: {err}")
    return True


def _open(path: str):
    if os.path.exists(path):
        return open(path, "rb")
    if os.path.exists(path + ".gz"):
        return gzip.open(path + ".gz", "rb")
    raise FileNotFoundError(path)


def read_idx(path: str) -> torch.Tensor:
    """Parse an idx-ubyte file (magic 0x0000 08 nd, big-endian dims, uint8 payload)."""
    with _open(path) as f:
        data = f.read()
    zero, dtype_code, nd = struct.unpack(">HBB", data[:4])
    if zero != 0 or dtype_code != 0x08:
        raise ValueError(f"{path}: not an unsigned-byte idx file (magic {data[:4].hex()})")
    dims = struct.unpack(">" + "I" * nd, data[4:4 + 4 * nd])
    n = 1
    for d in dims:
        n *= d
    payload = data[4 + 4 * nd:]
    if len(payload) != n:
        raise ValueError(f"{path}: payload has {len(payload)} bytes, header promises {n}")
    return torch.frombuffer(bytearray(payload), dtype=torch.uint8).view(*dims)


def write_idx(path: str, t: torch.Tensor) -> None:
    t = t.contiguous().to(torch.uint8)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(struct.pack(">HBB", 0, 0x08, t.dim()))
        f.write(struct.pack(">" + "I" * t.dim(), *t.shape))
        f.write(t.numpy().tobytes())


def synthesize_mnist_files(root: str, seed: int = 0, train: bool = True, n: Optional[int] = None) -> None:
    """Write deterministic synthetic idx files with MNIST's shape: each class is a blurred
    class-specific stroke pattern plus noise, so a ConvNet can actually learn it."""
    img_name, lbl_name, count = _FILES[train]
    n = count if n is None else n
    g = torch.Generator().manual_seed(seed + (0 if train else 1))
    labels = torch.randint(0, 10, (n,), generator=g)
    protos = torch.zeros(10, 28, 28)
    pg = torch.Generator().manual_seed(1234)
    for c in range(10):
        pts = torch.randint(4, 24, (6, 2), generator=pg)
        for (y, x) in pts.tolist():
            protos[c, y - 2:y + 3, x - 2:x + 3] += 1.0
    protos = (protos / protos.amax(dim=(1, 2), keepdim=True)).clamp(0, 1)
    noise = torch.rand(n, 28, 28, generator=g) * 0.25
    imgs = ((protos[labels] * 0.85 + noise).clamp(0, 1) * 255).to(torch.uint8)
    raw = os.path.join(root, "MNIST", "raw")
    write_idx(os.path.join(raw, img_name), imgs)
    write_idx(os.path.join(raw, lbl_name), labels.to(torch.uint8))


class MNIST:
    classes = [str(i) for i in range(10)]

    def __init__(self, root: str = "./data", train: bool = True, transform: Optional[Callable] = None,
                 target_transform: Optional[Callable] = None, download: bool = False,
                 synthetic_fallback: bool = False):
        self.root, self.train = root, train
        self.transform, self.target_transform = transform, target_transform
        img_name, lbl_name, _ = _FILES[train]
        raw = os.path.join(root, "MNIST", "raw")
        img_path, lbl_path = os.path.join(raw, img_name), os.path.join(raw, lbl_name)
        have = all(os.path.exists(p) or os.path.exists(p + ".gz") for p in (img_path, lbl_path))
        downloaded = download_mnist(root) if (download and not have) else False
        try:
            self.data = read_idx(img_path)
            self.targets = read_idx(lbl_path).to(torch.int64)
        except FileNotFoundError:
            if synthetic_fallback:
                synthesize_mnist_files(root, train=train)
                self.data = read_idx(img_path)
                self.targets = read_idx(lbl_path).to(torch.int64)
            else:
                hint = ("download=True was requested but no network is reachable from this machine; " if download and not downloaded else "")
                raise RuntimeError(
                    f"MNIST idx files not found under {raw}. {hint}Place the four *-ubyte[.gz] files there, "
                    "or pass synthetic_fallback=True / use data.SyntheticMNIST for shape-faithful synthetic data.")
        if self.data.dim() != 3 or self.data.shape[0] != self.targets.shape[0]:
            raise ValueError("MNIST: image/label files disagree")

    def __len__(self) -> int:
        return int(self.data.shape[0])

    def __getitem__(self, index: int) -> Tuple[torch.Tensor, int]:
        img = self.data[index].to(torch.float32).div_(255.0).unsqueeze(0)
        target = int(self.targets[index])
        if self.transform is not None:
            img = self.transform(img)
        if self.target_transform is not None:
            target = self.target_transform(target)
        return img, target

    def native_source(self):
        """Raw tensors for the C++ batch stager (``_C.BatchStager``): it gathers, applies ToTensor's 1/255 and pins
        without touching Python.  Only when no per-sample Python transform is in the way."""
        if self.transform is not None or self.target_transform is not None:
            return None
        return {"data": self.data, "targets": self.targets, "scale": 1.0 / 255.0, "sample_shape": (1,) + tuple(self.data.shape[1:])}

    def gather(self, indices: Sequence[int]):
        idx = torch.as_tensor(indices, dtype=torch.int64)
        imgs = self.data.index_select(0, idx).unsqueeze(1).to(torch.float32).div_(255.0)
        if self.transform is not None:
            imgs = torch.stack([self.transform(i) for i in imgs])
        tg = self.targets.index_select(0, idx)
        if self.target_transform is not None:
            tg = torch.as_tensor([self.target_transform(int(t)) for t in tg])
        return imgs, tg


class SyntheticMNIST:
    """In-memory synthetic data with MNIST's shapes and dtype — what the benchmarks use
    (BASELINE.json: "synthetic MNIST-shaped data ... there is no network")."""

    def __init__(self, n: int = 60000, seed: int = 0, num_classes: int = 10, image_shape=(1, 28, 28),
                 dtype=torch.float32):
        g = torch.Generator().manual_seed(seed)
        self.targets = torch.randint(0, num_classes, (n,), generator=g)
        self.data = torch.rand((n,) + tuple(image_shape), generator=g, dtype=torch.float32).to(dtype)

    def __len__(self):
        return int(self.data.shape[0])

    def __getitem__(self, i):
        return self.data[i], int(self.targets[i])

    def native_source(self):
        if self.data.dtype != torch.float32:
            return None
        return {"data": self.data, "targets": self.targets, "scale": 1.0, "sample_shape": tuple(self.data.shape[1:])}

    def gather(self, indices):
        idx = torch.as_tensor(indices, dtype=torch.int64)
        return self.data.index_select(0, idx), self.targets.index_select(0, idx)


class TensorDataset:
    def __init__(self, *tensors: torch.Tensor):
        if not tensors or any(t.shape[0] != tensors[0].shape[0] for t in tensors):
            raise ValueError("TensorDataset: tensors must share dim 0")
        self.tensors = tensors

    def __len__(self):
        return int(self.tensors[0].shape[0])

    def __getitem__(self, i):
        return tuple(t[i] for t in self.tensors)

    def gather(self, indices):
        idx = torch.as_tensor(indices, dtype=torch.int64)
        return tuple(t.index_select(0, idx) for t in self.tensors)
