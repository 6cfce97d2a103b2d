"""Model-based diffusion over the weights of an MNIST classifier — counterpart of upstream mbd/blackbox/mbd_mnist.py.

    python -m mbd_b200.blackbox.mbd_mnist --data_dir /tmp/jax_example_data/

The data is never downloaded: `data_dir` must hold the four files the reference caches (FILES).  Each step of the reference's
`reverse_once` is six launches (`mbd_mnist_step_launch`, csrc/mnist.cuh), captured once in a CUDA graph and replayed:
(1) Y0s = mean + noise * mask per tensor (add_noise_batch_to_params), (2) Js = mean over the step's minibatch of
log_softmax(MLP(x))[label] for every sample (layer 1 as one tensor-core GEMM over all samples), (3) the MPPI weights and
rew_hist[t] = Js.mean(), (4)-(5) the new mean sum_n w_n Y0s_n, (6) the train / test accuracy of the new mean.

Ported literally: the constants (Nsample = 256, Ndiffuse = 500, temp_sample = 0.3, betas = linspace(3e-5, 1e-3, 500)); the
stax init from PRNGKey(0) (init_params, [jax-recalled]); the key chain (`rng, Y0_rng = split(rng)`, `rng, batch_rng = split(rng)`
per step, the warm-up call at t = 0 discarding its carry); the per-tensor keys, noise (x 0.1 on W1) and Bernoulli(0.2) masks;
the minibatch `choice(batch_rng, 60000, (N,), replace=False)` = permutation(...)[:N] with two rounds of a stable sort of 32-bit
keys ([jax-recalled]).
Declared deviations:
  - the shared statistics kernel keeps MBD's guard std < 1e-4 -> 1;
  - the forward pass uses the project's fp32 functions and fixed summation orders (csrc/mnist.cuh) and layer 1 runs on the
    tensor cores in split TF32, so J is not XLA's bits; tests hold it to a float64 bound;
  - missing data files raise an error naming them and the directory searched.
One GPU.
"""
from __future__ import annotations

import gzip
import math
import os
import struct
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from mbd_b200 import _lib, ops, prng
from mbd_b200.planners.engine import LaunchInputs, StepEngine, make_schedule, pack_step_params

LAYERS = (784, 32, 32, 10)
HNU = 26506
FILES = ("train-images-idx3-ubyte.gz", "train-labels-idx1-ubyte.gz", "t10k-images-idx3-ubyte.gz", "t10k-labels-idx1-ubyte.gz")
# offsets of b1, W2, b2, W3, b3 in a parameter row; W1 is stored transposed, [32][784], at offset 0
OFF_B1 = 784 * 32
OFF_W2 = OFF_B1 + 32
OFF_B2 = OFF_W2 + 32 * 32
OFF_W3 = OFF_B2 + 32
OFF_B3 = OFF_W3 + 32 * 10


@dataclass
class Args:
    Nsample: int = 256
    Ndiffuse: int = 500
    temp_sample: float = 0.3
    beta0: float = 3e-5
    betaT: float = 1e-3
    seed: int = 0
    data_dir: str = "/tmp/jax_example_data/"
    eval_every: int = 1
    log_every: int = 1


# ---- data ------------------------------------------------------------------------------------------------------------------
def read_idx(path: str, magic: int) -> np.ndarray:
    """one gzip-compressed IDX file (2049: labels, 2051: images); checks the magic number and that the payload holds exactly
    the items the header announces"""
    with gzip.open(path, "rb") as fh:
        data = fh.read()
    ndim = 1 if magic == 2049 else 3
    if len(data) < 4 + 4 * ndim:
        raise ValueError(f"{path}: truncated IDX header")
    got = struct.unpack(">I", data[:4])[0]
    if got != magic:
        raise ValueError(f"{path}: magic number {got}, expected {magic}")
    dims = struct.unpack(">" + "I" * ndim, data[4:4 + 4 * ndim])
    body = data[4 + 4 * ndim:]
    if len(body) != int(np.prod(dims)):
        raise ValueError(f"{path}: {len(body)} payload bytes, the header announces {int(np.prod(dims))}")
    return np.frombuffer(body, np.uint8).reshape(dims)


def load_mnist(data_dir: str):
    """(train_x [n, 784] uint8, train_y [n] uint8, test_x, test_y) from the four files of FILES in data_dir"""
    paths = [os.path.join(data_dir, f) for f in FILES]
    missing = [f for f, p in zip(FILES, paths) if not os.path.isfile(p)]
    if missing:
        raise FileNotFoundError(f"MNIST files missing from {os.path.abspath(data_dir)}: {', '.join(missing)} "
                                f"(this port never downloads; it needs {', '.join(FILES)})")
    out = []
    for k in range(2):
        x = read_idx(paths[2 * k], 2051)
        y = read_idx(paths[2 * k + 1], 2049)
        if x.shape[1:] != (28, 28):
            raise ValueError(f"{paths[2 * k]}: images are {x.shape[1:]}, expected (28, 28)")
        if x.shape[0] != y.shape[0]:
            raise ValueError(f"{paths[2 * k]}: {x.shape[0]} images but {y.shape[0]} labels")
        if y.size and int(y.max()) > 9:
            raise ValueError(f"{paths[2 * k + 1]}: label {int(y.max())} out of 0..9")
        out += [np.ascontiguousarray(x.reshape(x.shape[0], 784)), np.ascontiguousarray(y)]
    return tuple(out)


# ---- host PRNG (init only) ---------------------------------------------------------------------------------------------------
def _fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _logf(x):
    """include/mbd_fp32.h mbd_logf, elementwise in numpy (fma as one float64 rounding)"""
    f = np.float32
    u = x.astype(np.float32).view(np.uint32)
    e = (u >> np.uint32(23)).astype(np.int32) - 127
    m = ((u & np.uint32(0x007FFFFF)) | np.uint32(0x3F800000)).view(np.float32)
    big = m > f(1.41421354)
    m = np.where(big, m * f(0.5), m).astype(f)
    e = np.where(big, e + 1, e)
    fr = (m - f(1.0)).astype(f)
    p = np.full_like(fr, f(-8.101639897e-02))
    for c in (1.271235049e-01, -1.297222823e-01, 1.420216709e-01, -1.664224863e-01, 2.000146955e-01, -2.500029802e-01, 3.333332837e-01):
        p = _fma32(p, fr, np.full_like(fr, f(c)))
    f2 = (fr * fr).astype(f)
    fe = e.astype(f)
    r = _fma32((p * fr).astype(f), f2, (fe * f(-2.12194440e-4)).astype(f))
    r = _fma32(np.full_like(fr, f(-0.5)), f2, r)
    r = (fr + r).astype(f)
    return _fma32(fe, np.full_like(fr, f(0.693359375)), r)


def _erfinv(x):
    """include/mbd_fp32.h mbd_erfinvf (Giles' single-precision polynomial, XLA's f32 ErfInv)"""
    f = np.float32
    x = x.astype(f)
    w = -_logf(((f(1.0) - x) * (f(1.0) + x)).astype(f))
    lo = w < f(5.0)
    w1 = (w - f(2.5)).astype(f)
    w2 = (np.sqrt(w.astype(np.float64)).astype(f) - f(3.0)).astype(f)
    c1 = (2.81022636e-08, 3.43273939e-07, -3.5233877e-06, -4.39150654e-06, 0.00021858087, -0.00125372503, -0.00417768164,
          0.246640727, 1.50140941)
    c2 = (-0.000200214257, 0.000100950558, 0.00134934322, -0.00367342844, 0.00573950773, -0.0076224613, 0.00943887047,
          1.00167406, 2.83297682)
    ww = np.where(lo, w1, w2).astype(f)
    p = np.where(lo, f(c1[0]), f(c2[0])).astype(f)
    for a, b in zip(c1[1:], c2[1:]):
        p = _fma32(p, ww, np.where(lo, f(a), f(b)).astype(f))
    return (p * x).astype(f)


def _unit(bits):
    return ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)


def normal_host(key, shape) -> np.ndarray:
    """jax.random.normal(key, shape) (f32) on the host, with the project's erfinv"""
    f = np.float32
    n = int(np.prod(shape))
    u = (_unit(prng.random_bits(key, n)) * f(2.0) + f(-0.99999994)).astype(f)
    u = np.maximum(u, f(-0.99999994))
    return (f(1.41421354) * _erfinv(u)).astype(f).reshape(shape)


def truncated_normal_host(key, lower: float, upper: float, shape) -> np.ndarray:
    """jax.random.truncated_normal(key, lower, upper, shape) (f32) **[jax-recalled]**: u = uniform(key, shape, minval=erf(lower /
    sqrt2), maxval=erf(upper / sqrt2)), out = sqrt2 * erf_inv(u), clipped to the open interval"""
    f = np.float32
    sqrt2 = f(np.sqrt(2.0))
    a = f(math.erf(float(f(lower) / sqrt2)))
    b = f(math.erf(float(f(upper) / sqrt2)))
    n = int(np.prod(shape))
    u = np.maximum(a, (_unit(prng.random_bits(key, n)) * (b - a) + a).astype(f))
    out = (sqrt2 * _erfinv(u)).astype(f)
    return np.clip(out, np.nextafter(f(lower), f(np.inf)), np.nextafter(f(upper), f(-np.inf))).reshape(shape)


def init_params(seed: int = 0):
    """stax.serial(Dense(32), Relu, Dense(32), Relu, Dense(10), LogSoftmax) initialised with PRNGKey(seed) **[jax-recalled]**:
    serial splits `rng, layer_rng = split(rng)` once per layer; Dense splits k1, k2 and draws W = glorot_normal(k1, (in, out)),
    b = normal(k2, (out,)) * 1e-2.  Returns [(W1, b1), (W2, b2), (W3, b3)] in the reference's (in, out) layout."""
    f = np.float32
    rng = prng.PRNGKey(seed)
    params = []
    for layer in range(6):
        rng, layer_rng = prng.split2(rng)
        if layer % 2:
            continue
        fin, fout = LAYERS[layer // 2], LAYERS[layer // 2 + 1]
        k1, k2 = prng.split(layer_rng)
        std = f(np.sqrt(f(1.0) / f((fin + fout) / 2.0))) / f(0.87962566103423978)
        W = (truncated_normal_host(k1, -2.0, 2.0, (fin, fout)) * std).astype(f)
        b = (normal_host(k2, (fout,)) * f(1e-2)).astype(f)
        params.append((W, b))
    return params


def params_to_row(params) -> np.ndarray:
    """the device row of a parameter set: W1 transposed, b1, W2, b2, W3, b3"""
    (W1, b1), (W2, b2), (W3, b3) = params
    return np.concatenate([np.asarray(W1, np.float32).T.reshape(-1), b1, np.asarray(W2).reshape(-1), b2,
                           np.asarray(W3).reshape(-1), b3]).astype(np.float32)


def row_to_params(row):
    """inverse of params_to_row: [(W1, b1), (W2, b2), (W3, b3)] in (in, out) layout"""
    row = np.asarray(row, np.float32)
    return [(row[:OFF_B1].reshape(32, 784).T.copy(), row[OFF_B1:OFF_W2].copy()),
            (row[OFF_W2:OFF_B2].reshape(32, 32).copy(), row[OFF_B2:OFF_W3].copy()),
            (row[OFF_W3:OFF_B3].reshape(32, 10).copy(), row[OFF_B3:].copy())]


def step_keys(seed: int, Ndiffuse: int):
    """(keys [Ndiffuse, 12, 2], sub [Ndiffuse, 2, 2]) uint32: row t = the (noise, mask) keys of W1, b1, W2, b2, W3, b3 of step t
    (from Y0_rng: `k, kn = split(k)`, `k, ku = split(k)` per tensor) and the two permutation round keys of its minibatch (from
    batch_rng: `key, sub = split(key)` per round); the chain is `rng = PRNGKey(seed)`, then per step t = Ndiffuse - 1 ... 1
    `rng, Y0_rng = split(rng)` and `rng, batch_rng = split(rng)`"""
    keys = np.zeros((Ndiffuse, 12, 2), np.uint32)
    sub = np.zeros((Ndiffuse, 2, 2), np.uint32)
    rng = prng.PRNGKey(seed)
    for t in range(Ndiffuse - 1, 0, -1):
        rng, k = prng.split2(rng)
        for q in range(6):
            k, keys[t, 2 * q] = prng.split2(k)
            k, keys[t, 2 * q + 1] = prng.split2(k)
        rng, kb = prng.split2(rng)
        for r in range(2):
            kb, sub[t, r] = prng.split2(kb)
    return keys, sub


# ---- device engine -----------------------------------------------------------------------------------------------------------
class MnistEngine(StepEngine):
    """One MNIST solve (B = 1, H = 1, HNu = 26506) stepped by `mbd_mnist_step_launch`; the solve-level surface of
    StepEngine (set_step, step, capture, check_exchange, solve).  Ybars[0][t] = the mean before step t (row Ndiffuse - 1 =
    the init), rew_hist[0][t] = Js.mean() of step t, acc_hist[t] = train / test correct-counts of the mean after step t (-1
    where not evaluated)."""

    def __init__(self, data, Nsample: int, temp: float, Ndiffuse: int, eval_every: int = 1, device: Optional[torch.device] = None):
        train_x, train_y, test_x, test_y = data
        if not 1 <= int(Nsample) <= len(train_x):
            raise ValueError(f"Nsample must lie in 1 .. {len(train_x)} (the minibatch has Nsample images)")
        # launch (3) reads the plan's temperature
        super().__init__(LaunchInputs.none(), Nsample, 1, HNU, Ndiffuse, False, B=1, temp=temp, device=device)
        d = self.device
        u8 = lambda a: torch.from_numpy(np.array(a, np.uint8, copy=True)).to(d)   # noqa: E731
        self.train_x, self.train_y, self.test_x, self.test_y = u8(train_x), u8(train_y), u8(test_x), u8(test_y)
        self.n_train, self.n_test = len(train_x), len(test_x)
        self.keys = torch.zeros((self.Nd, 12, 2), device=d, dtype=torch.int32)
        self.batch_idx = torch.zeros((self.Nd, self.N), device=d, dtype=torch.int32)
        self.acc_hist = torch.full((self.Nd, 2), -1, device=d, dtype=torch.int32)
        self.eval_every = int(eval_every)
        self._bufs = _lib.MnistBufs(self.train_x.data_ptr(), self.train_y.data_ptr(), self.test_x.data_ptr(), self.test_y.data_ptr(),
                                    self.keys.data_ptr(), self.batch_idx.data_ptr(), self.acc_hist.data_ptr(), LAYERS,
                                    self.n_train, self.n_test, self.eval_every)

    def load_schedule(self, seed: int, sigmas, init_row):
        """uploads the solve: the keys of every step, sigmas, the minibatch table (computed on the device) and the init row"""
        if len(sigmas) != self.Nd:
            raise ops.MbdError(f"schedule of {len(sigmas)} steps does not match the engine (Ndiffuse={self.Nd})")
        keys, sub = step_keys(seed, self.Nd)
        self.params[0].copy_(torch.from_numpy(pack_step_params(np.zeros((self.Nd, 2), np.uint32), sigmas, None, None)))
        self.keys.copy_(torch.from_numpy(keys.view(np.int32)))
        ops.mnist_batch_indices(sub, self.Nd, self.n_train, self.N, self.batch_idx)
        self.Ybars[0, self.Nd - 1].copy_(torch.from_numpy(np.asarray(init_row, np.float32)))
        self.acc_hist.fill_(-1)

    def set_step(self, i: int):
        """step counter <- i, and clears the control block's error word: a reloaded or re-armed solve must not inherit the
        past-the-end flag of an earlier run (the accuracy launch writes nothing while it is set)"""
        super().set_step(i)
        self.ctl[:, 2].zero_()

    def _launch(self):
        ops.mnist_step_launch(self._plan_c, self.Nd, self._bufs)

    def forward(self, Y0s: torch.Tensor, rows: torch.Tensor, z1: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Js of the parameter rows Y0s [n, 26506] on the training images `rows` (test entry point)"""
        Js = torch.empty(Y0s.shape[0], device=self.device)
        ops.mnist_forward(Y0s, self._bufs, rows, Js, z1)
        return Js


def run_mnist(args: Args, data=None, progress: bool = False):
    """the reference's solve.  Returns dict(J [Ndiffuse - 1] = Js.mean() of steps Ndiffuse - 1 ... 1, train_acc / test_acc
    [Ndiffuse - 1] (NaN where not evaluated), params = the final [(W, b)] in (in, out) layout)."""
    data = load_mnist(args.data_dir) if data is None else data
    eng = MnistEngine(data, args.Nsample, args.temp_sample, args.Ndiffuse, args.eval_every)
    sigmas = make_schedule(args.beta0, args.betaT, args.Ndiffuse)[3]
    eng.load_schedule(args.seed, sigmas, params_to_row(init_params(args.seed)))

    def log(t):
        acc = eng.acc_hist[t].cpu().numpy()
        print(f"step {t}: J={eng.rew_hist[0, t].item():.2f}, train_acc={acc[0] / eng.n_train:.3f}, "
              f"test_acc={acc[1] / eng.n_test:.3f}", flush=True)
    # the warm-up step of the capture is re-run from the same state; launch (1) re-zeroes the counts it adds to
    eng.solve(log if progress else None, args.log_every)
    acc = eng.acc_hist[1:].flip(0).cpu().numpy().astype(np.float64)
    acc[acc < 0] = np.nan
    return dict(J=eng.rew_hist[0, 1:].flip(0).cpu().numpy(), train_acc=acc[:, 0] / eng.n_train, test_acc=acc[:, 1] / eng.n_test,
                params=row_to_params(eng.Ybars[0, 0].cpu().numpy()))


def main(argv=None):
    import tyro
    args = tyro.cli(Args, args=argv)
    res = run_mnist(args, progress=True)
    print(f"MNIST MBD: J {res['J'][0]:.3f} -> {res['J'][-1]:.3f}; final train_acc {res['train_acc'][-1]:.4f}, "
          f"test_acc {res['test_acc'][-1]:.4f}")
    return res


if __name__ == "__main__":
    main()
