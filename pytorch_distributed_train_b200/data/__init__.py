"""Input pipeline: samplers, DataLoader, MNIST (idx parser), synthetic datasets, MixUp, CutMix, random affine and elastic
augmentation."""
from .augment import RandomAffine
from .dataloader import DataLoader, DevicePrefetcher, default_collate
from .elastic import ElasticTransform
from .mix import CutMix, MixUp
from .mixup import mixup
from .mnist import MNIST, SyntheticMNIST, TensorDataset, read_idx, synthesize_mnist_files, write_idx
from .sampler import BatchSampler, DistributedSampler, RandomSampler, Sampler, SequentialSampler

__all__ = [
    "DataLoader", "DevicePrefetcher", "default_collate", "MNIST", "SyntheticMNIST", "TensorDataset",
    "read_idx", "write_idx", "synthesize_mnist_files", "BatchSampler", "DistributedSampler",
    "RandomSampler", "Sampler", "SequentialSampler", "mixup", "RandomAffine", "ElasticTransform", "MixUp",
    "CutMix",
]
