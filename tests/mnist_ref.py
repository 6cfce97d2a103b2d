"""Host restatements of one MNIST step (csrc/mnist.cuh) and a float64 forward pass with a running error radius.

Sampling and the minibatch are JAX's bits, so they are restated exactly: the noise with the oracle's normal (the same fp32
spec as the device), the masks and permutation keys with mbd_b200.prng.  The forward pass is evaluated in float64 and every
fp32 result of the device gets a radius built from:
  - u = 2^-24 per fp32 operation (recursive sums: gamma_n = n u / (1 - n u) times the sum of magnitudes);
  - the split-TF32 weight: |w - hi - lo| <= 2^-22 |w| (two round-to-nearest TF32 roundings, 10 explicit mantissa bits each);
  - the tensor-core accumulation of one K tile: TC_ACC per accumulation (33 per tile: 32 products onto a zero) times the sum
    of magnitudes.  This constant is ASSUMED, NOT PROVEN: the PTX ISA does not specify the rounding of wgmma's fp32
    accumulation; 2u per accumulation (truncation instead of rounding) is assumed.  What the device does is measured by
    tests/test_mnist_gpu.py::test_z1_error_measured (the largest |Z1_device - Z1_64| / (sum_k |p_k w_k| / 255)), which is
    recorded in DESIGN.md §5d and must stay below the assumed budget;
  - EXP_REL / LOG_ABS: the measured accuracy of mbd_expf / mbd_logf (tests/test_fp32_spec.py holds them to 4 ulp)."""
import numpy as np

from mbd_b200 import prng
from mbd_b200.blackbox import mbd_mnist as mm

f32 = np.float32
U = 2.0 ** -24
SPLIT = 2.0 ** -22
TC_ACC = 2 * U
EXP_REL = 4 * 2.0 ** -23
LOG_ABS = 4 * 2.0 ** -23
SIZES = (784 * 32, 32, 32 * 32, 32, 32 * 10, 10)
OFFS = (0, mm.OFF_B1, mm.OFF_W2, mm.OFF_B2, mm.OFF_W3, mm.OFF_B3)


def gamma(n):
    return n * U / (1 - n * U)


def _unit(bits):
    return ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - f32(1.0)


def sample(orc, keys_t, sigma, mean_row, N):
    """Y0s [N, 26506] of add_noise_batch_to_params: per tensor, noise = normal(kn, (N,) + shape) * sigma (* 0.1 on W1), mask =
    uniform(ku, (N,) + shape) < 0.2, Y = mean + noise * mask; W1 is drawn in JAX's (n, in, out) order and stored transposed"""
    mean_row = np.asarray(mean_row, f32)
    out = np.empty((N, mm.HNU), f32)
    for t in range(6):
        kn, ku = np.asarray(keys_t[2 * t], np.uint32), np.asarray(keys_t[2 * t + 1], np.uint32)
        noise = (orc.normal(kn, (N * SIZES[t],)) * f32(sigma)).astype(f32)
        if t == 0:
            noise = (noise * f32(0.1)).astype(f32)
        mask = (_unit(prng.random_bits(ku, N * SIZES[t])) < f32(0.2)).astype(f32)
        d = (noise * mask).astype(f32).reshape(N, SIZES[t])
        if t == 0:
            d = d.reshape(N, 784, 32).transpose(0, 2, 1).reshape(N, SIZES[0])
        out[:, OFFS[t]:OFFS[t] + SIZES[t]] = (mean_row[None, OFFS[t]:OFFS[t] + SIZES[t]] + d).astype(f32)
    return out


def batch_indices(sub_t, n_data, N):
    """choice(batch_rng, n_data, (N,), replace=False) = permutation(batch_rng, n_data)[:N] [jax-recalled]: two rounds of a
    stable sort of arange by random_bits(sub_r, (n_data,))"""
    x = np.arange(n_data, dtype=np.int32)
    for r in range(2):
        keys = prng.random_bits(np.asarray(sub_t[r], np.uint32), n_data)
        x = x[np.argsort(keys, kind="stable")]
    return x[:N]


def forward64(row, X, Y, tf32_single=False, slip=None):
    """float64 forward of one parameter row on images X [M, 784] (uint8) and labels Y [M].  Returns dict(J, rJ = radius of the
    device's fp32 J, z1 [M, 32] (before b1), rz1, lp [M, 10], rlp [M] (radius of every lp entry of an image)).
    tf32_single / slip restate a deliberately wrong kernel (tests of the radius): 'no255', 'norelu', 'nob2'."""
    (W1, b1), (W2, b2), (W3, b3) = [(np.asarray(W, np.float64), np.asarray(b, np.float64)) for W, b in mm.row_to_params(row)]
    if tf32_single:
        W1 = _tf32(np.asarray(mm.row_to_params(row)[0][0], f32)).astype(np.float64)
    p = np.asarray(X, np.float64)
    s1 = p @ W1
    S1 = p @ np.abs(W1)
    z1 = s1 / (1.0 if slip == "no255" else 255.0)
    rz1 = (SPLIT + TC_ACC * 33 + gamma(49)) * S1 / 255.0 + U * np.abs(z1)
    a1 = z1 + b1
    h1 = a1 if slip == "norelu" else np.maximum(a1, 0.0)
    rh1 = rz1 + U * np.abs(a1)
    z2 = h1 @ W2 + (0.0 if slip == "nob2" else b2)
    rz2 = rh1 @ np.abs(W2) + gamma(33) * (np.abs(h1) @ np.abs(W2) + np.abs(b2)) + U * np.abs(z2)
    h2 = np.maximum(z2, 0.0)
    z3 = h2 @ W3 + b3
    rz3 = rz2 @ np.abs(W3) + gamma(33) * (np.abs(h2) @ np.abs(W3) + np.abs(b3))
    mx = z3.max(1, keepdims=True)
    s = z3 - mx
    se = np.exp(s).sum(1, keepdims=True)
    lse = np.log(se)
    lp = s - lse
    ez = rz3.max(1)
    # lp_c = (z_c - mx) - lse: the inputs move each term by <= 2 ez (lse is 1-Lipschitz in the max norm); the roundings of the
    # subtractions, the exps, the 10-term sum and the log add the rest
    rlp = 2 * ez + 2 * ez + U * np.abs(s).max(1) + (EXP_REL + gamma(10)) * 1.0 + LOG_ABS * np.maximum(1.0, np.abs(lse[:, 0])) \
        + U * np.abs(lp).max(1)
    v = lp[np.arange(len(Y)), np.asarray(Y, np.int64)]
    M = len(Y)
    depth = (M + 255) // 256 + 8
    J = v.mean()
    rJ = rlp.mean() + gamma(depth) * np.abs(v).mean() + U * abs(J)
    return dict(J=J, rJ=rJ, z1=z1, rz1=rz1, S1=S1, lp=lp, rlp=rlp)


def _tf32(x):
    """round-to-nearest-even to TF32 (10 explicit mantissa bits)"""
    u = np.asarray(x, f32).view(np.uint32).astype(np.uint64)
    u = (u + 0xFFF + ((u >> 13) & 1)) & ~np.uint64(0x1FFF)
    return u.astype(np.uint32).view(f32)


def accuracy_bounds(row, X, Y):
    """(certain, undecided) correct-counts: certain = images whose label is the float64 argmax by more than the radius of the two
    entries; undecided = images whose label is within the radius of the top value (either answer is possible)"""
    r = forward64(row, X, Y)
    lp, rad = r["lp"], r["rlp"]
    lab = lp[np.arange(len(Y)), np.asarray(Y, np.int64)]
    other = lp.copy()
    other[np.arange(len(Y)), np.asarray(Y, np.int64)] = -np.inf
    top_other = other.max(1)
    certain = lab - top_other > 2 * rad
    undecided = np.abs(lab - top_other) <= 2 * rad
    return int(certain.sum()), int(undecided.sum())
