"""Read the reference-generated fixtures under tests/golden: a file's arrays, and the flat indices of the gradient entries
a training fixture samples per parameter (make_golden.py's `gsamp::<name>`).  Imports nothing from the reference, so GPU
tests can use it."""
import os
import zlib

import numpy as np
import torch

from conftest import GOLDEN

N_GRAD_SAMPLES = 32


def load(name: str) -> dict:
    return dict(np.load(os.path.join(GOLDEN, name), allow_pickle=False))


def grad_sample_index(name: str, numel: int) -> torch.Tensor:
    """N_GRAD_SAMPLES flat indices into parameter `name`'s gradient, seeded by the name."""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randint(0, numel, (N_GRAD_SAMPLES,), generator=g)
