"""A synthetic dataset with MNIST's shapes and file format: 60 000 / 10 000 28x28 uint8 images made of ten class templates plus
noise (so a classifier can learn it), written as the four gzip IDX files the reference caches."""
import gzip
import os
import struct

import numpy as np

from mbd_b200.blackbox import mbd_mnist


def write_idx(path: str, arr: np.ndarray, magic: int = None, count: int = None):
    """gzip IDX file of a uint8 array (magic 2049 for 1-d labels, 2051 for 3-d images); `count` overrides the item count of the
    header (to build a mismatched file)"""
    arr = np.ascontiguousarray(arr, np.uint8)
    magic = (2049 if arr.ndim == 1 else 2051) if magic is None else magic
    dims = list(arr.shape)
    if count is not None:
        dims[0] = count
    with gzip.open(path, "wb") as fh:
        fh.write(struct.pack(">I", magic) + struct.pack(">" + "I" * arr.ndim, *dims) + arr.tobytes())


def make(n_train: int = 60000, n_test: int = 10000, seed: int = 0):
    """(train_x [n, 784], train_y [n], test_x, test_y) uint8: image = clip(template[label] + noise) with per-class templates of
    random strokes and noise of std 60"""
    r = np.random.default_rng(seed)
    tmpl = np.zeros((10, 28, 28), np.float32)
    for c in range(10):
        for _ in range(6):
            y0, x0 = r.integers(4, 24, 2)
            h, w = r.integers(2, 10, 2)
            tmpl[c, y0:y0 + h, x0:x0 + w] = 220.0
    tmpl = tmpl.reshape(10, 784)

    def draw(n):
        y = r.integers(0, 10, n).astype(np.uint8)
        x = np.clip(tmpl[y] + r.normal(0.0, 60.0, (n, 784)).astype(np.float32), 0, 255).astype(np.uint8)
        return x, y

    trx, trY = draw(n_train)
    tex, teY = draw(n_test)
    return trx, trY, tex, teY


def write_dir(d: str, data):
    """the four files of mbd_mnist.FILES in directory d"""
    trx, trY, tex, teY = data
    os.makedirs(d, exist_ok=True)
    for name, a in zip(mbd_mnist.FILES, (trx.reshape(-1, 28, 28), trY, tex.reshape(-1, 28, 28), teY)):
        write_idx(os.path.join(d, name), a)
