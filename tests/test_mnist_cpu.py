"""MNIST solve, host side: the IDX parser, the stax init, the key / noise / mask / minibatch restatements, the float64 forward's
radius against deliberate slips, and the entry points' argument checks (which run before any CUDA call)."""
import ctypes
import os

import numpy as np
import pytest

from mbd_b200 import _lib, prng
from mbd_b200.blackbox import mbd_mnist as mm
from tests import mnist_ref as mr
from tests import mnist_synth as ms

f32 = np.float32


def test_idx_round_trip_and_rejections(tmp_path):
    data = ms.make(300, 50)
    ms.write_dir(str(tmp_path), data)
    got = mm.load_mnist(str(tmp_path))
    for a, b in zip(got, data):
        assert np.array_equal(a, b)
    p = str(tmp_path / "bad.gz")
    ms.write_idx(p, data[1], magic=2051)
    with pytest.raises(ValueError, match="magic"):
        mm.read_idx(p, 2049)
    ms.write_idx(p, data[1], count=301)
    with pytest.raises(ValueError, match="payload"):
        mm.read_idx(p, 2049)
    import gzip
    with gzip.open(p, "wb") as fh:
        fh.write(b"\x00\x00\x08")
    with pytest.raises(ValueError, match="truncated"):
        mm.read_idx(p, 2049)
    ms.write_idx(str(tmp_path / mm.FILES[1]), data[1][:299])
    with pytest.raises(ValueError, match="labels"):
        mm.load_mnist(str(tmp_path))


def test_missing_data_dir_names_the_files(tmp_path):
    with pytest.raises(FileNotFoundError) as ei:
        mm.load_mnist(str(tmp_path / "nowhere"))
    msg = str(ei.value)
    assert "nowhere" in msg and all(f in msg for f in mm.FILES)


def test_init_shapes_std_and_truncation():
    params = mm.init_params(0)
    assert [(W.shape, b.shape) for W, b in params] == [((784, 32), (32,)), ((32, 32), (32,)), ((32, 10), (10,))]
    for (W, b), (fin, fout) in zip(params, ((784, 32), (32, 32), (32, 10))):
        sd = np.sqrt(2.0 / (fin + fout))
        # glorot_normal: truncated at +-2 of the unit normal, rescaled so the std is sqrt(2 / (in + out))
        assert np.abs(W).max() <= 2 * sd / 0.87962566103423978 * (1 + 1e-6)
        if W.size > 1000:
            assert abs(W.std() / sd - 1) < 0.05
        assert np.abs(b).max() < 0.05 and b.dtype == f32
    row = mm.params_to_row(params)
    assert row.shape == (mm.HNU,)
    for (a, b), (c, d) in zip(params, mm.row_to_params(row)):
        assert np.array_equal(a, c) and np.array_equal(b, d)


@pytest.mark.parametrize("part", [False, True])
def test_keys_noise_and_minibatch_restatements(orc, part):
    prng.set_layout(part)
    orc.set_prng_layout(part)
    try:
        keys, sub = mm.step_keys(0, 5)
        rng = prng.PRNGKey(0)
        for t in (4, 3):
            rng, y0 = prng.split2(rng)
            k = y0
            for q in range(6):
                k, kn = prng.split(k)
                k, ku = prng.split(k)
                assert np.array_equal(keys[t, 2 * q], kn) and np.array_equal(keys[t, 2 * q + 1], ku)
            rng, kb = prng.split2(rng)
            kb, s0 = prng.split(kb)
            assert np.array_equal(sub[t, 0], s0)
        assert not keys[0].any()
        # the host normal (init) agrees with the oracle's (the device spec)
        k0 = keys[4, 0]
        assert np.abs(mm.normal_host(k0, (4096,)) - orc.normal(k0, (4096,))).max() <= 2e-7 * 4
        # a small sample: W1 entries follow JAX's (n, in, out) counters, masks are ~20 %, b-noise has std sigma
        Y = mr.sample(orc, keys[4], 0.5, np.zeros(mm.HNU, f32), 3)
        W1 = Y[:, :mm.OFF_B1].reshape(3, 32, 784).transpose(0, 2, 1).reshape(-1)
        n = orc.normal(keys[4, 0], (3 * 784 * 32,)) * f32(0.5) * f32(0.1)
        nz = W1 != 0
        assert np.array_equal(W1[nz], n.astype(f32)[nz]) and abs(nz.mean() - 0.2) < 0.01
        # choice = two stable sorts; ties keep index order
        idx = mr.batch_indices(sub[4], 60000, 256)
        assert len(np.unique(idx)) == 256 and idx.min() >= 0 and idx.max() < 60000
        bits = prng.random_bits(sub[4, 0], 60000)
        assert np.array_equal(np.arange(60000)[np.argsort(bits, kind="stable")][:5],
                              sorted(range(60000), key=lambda i: (int(bits[i]), i))[:5])
    finally:
        prng.set_layout(False)
        orc.set_prng_layout(False)


def _mirror(row, X, Y, tf32_single=False, slip=None):
    """fp32 forward in the device's orders (numpy), with deliberate slips of the forward pass: 'w1_x10' (layer-1 weights ten
    times too large), 'no255' (pixels not divided by 255), 'norelu' (layer-1 ReLU dropped), 'nob2' (b2 omitted).  The sampling
    slips (the 0.1 on W1's noise, the mask probability) are caught by the device's bit-for-bit Y0s test instead."""
    (W1, b1), (W2, b2), (W3, b3) = mm.row_to_params(row)
    if slip == "w1_x10":
        W1 = (W1 * f32(10.0)).astype(f32)
    W1u = mr._tf32(W1) if tf32_single else W1
    p = np.asarray(X, np.float64)
    z1 = (p @ W1u.astype(np.float64)).astype(f32)
    if slip != "no255":
        z1 = (z1 / f32(255.0)).astype(f32)
    a1 = (z1 + b1).astype(f32)
    h1 = a1 if slip == "norelu" else np.maximum(a1, f32(0))
    z2 = np.zeros((len(X), 32), f32)
    for k in range(32):
        z2 = (z2 + (h1[:, k:k + 1] * W2[k][None]).astype(f32)).astype(f32)
    if slip != "nob2":
        z2 = (z2 + b2).astype(f32)
    h2 = np.maximum(z2, f32(0))
    z3 = np.zeros((len(X), 10), f32)
    for k in range(32):
        z3 = (z3 + (h2[:, k:k + 1] * W3[k][None]).astype(f32)).astype(f32)
    z3 = (z3 + b3).astype(f32)
    s = (z3 - z3.max(1, keepdims=True)).astype(f32)
    lse = np.log(np.exp(s.astype(np.float64)).sum(1)).astype(f32)
    lp = (s - lse[:, None]).astype(f32)
    return float(np.float32(lp[np.arange(len(Y)), Y].astype(f32).sum(dtype=f32) / f32(len(Y))))


@pytest.mark.parametrize("slip", [None, "w1_x10", "no255", "norelu", "nob2"])
def test_radius_against_slips(slip):
    """an fp32 mirror stays within the float64 radius of J on constructed parameter sets; each slip leaves it"""
    rng = np.random.default_rng(3)
    data = ms.make(256, 10, seed=3)
    X, Y = data[0], data[1].astype(np.int64)
    init = mm.params_to_row(mm.init_params(0))
    left = 0
    for k in range(6):
        row = (init + rng.normal(0, 0.02, mm.HNU)).astype(f32)
        row[mm.OFF_B1:mm.OFF_W2] = rng.normal(0.3, 0.5, 32).astype(f32)   # some units dead, some alive
        row[mm.OFF_B2:mm.OFF_W3] = rng.normal(0.5, 0.5, 32).astype(f32)
        r = mr.forward64(row, X, Y)
        got = _mirror(row, X, Y, slip=slip)
        left += abs(got - r["J"]) > r["rJ"]
    if slip is None:
        assert left == 0
    else:
        assert left >= 5, f"slip {slip} stayed inside the radius on {6 - left} of 6 parameter sets"


def test_single_pass_tf32_leaves_the_z1_radius():
    """single-pass TF32 on W1 moves the layer-1 pre-activations outside their radius: the split is needed to stay inside it.
    (The mean over the minibatch in J averages this error down below J's radius, so the check is on Z1, which the device
    also returns.)"""
    rng = np.random.default_rng(4)
    X, Y = ms.make(256, 10, seed=4)[:2]
    row = (mm.params_to_row(mm.init_params(0)) + rng.normal(0, 0.02, mm.HNU)).astype(f32)
    r = mr.forward64(row, X, Y)
    W1 = mm.row_to_params(row)[0][0]
    z_single = (np.asarray(X, np.float64) @ mr._tf32(W1).astype(np.float64)) / 255.0
    z_split = (np.asarray(X, np.float64) @ W1.astype(np.float64)) / 255.0
    assert (np.abs(z_split - r["z1"]) <= r["rz1"]).all()
    assert (np.abs(z_single - r["z1"]) > r["rz1"]).mean() > 0.5


def test_c_restatement_within_the_radius():
    """the C restatement of the SIMT remainder, fed the float64 Z1 rounded to fp32, stays within J's float64 radius"""
    from tests import mnist_oracle as mo
    rng = np.random.default_rng(5)
    X, Y = ms.make(300, 10, seed=5)[:2]
    init = mm.params_to_row(mm.init_params(0))
    rows = (init[None] + rng.normal(0, 0.03, (4, mm.HNU))).astype(f32)
    rs = [mr.forward64(r, X, Y) for r in rows]
    J = mo.js_from_z1(rows, np.stack([r["z1"] for r in rs]).astype(f32), Y)
    for j, r in zip(J, rs):
        assert abs(float(j) - r["J"]) <= r["rJ"]


def test_argument_rejection():
    L = _lib.lib()
    plan = _lib.StepPlan()
    plan.H, plan.nu, plan.n_total, plan.n_local, plan.P = 1, mm.HNU, 256, 256, 1
    dummy = 0x1000
    for f in ("params_dev", "ctl_dev", "Ybars_dev", "Y0s_dev", "rews_dev", "rews_all_dev", "logp_dev", "weights_dev", "runs_dev",
              "scalars_dev"):
        setattr(plan, f, dummy)

    def bufs(**kw):
        b = _lib.MnistBufs(dummy, dummy, dummy, dummy, dummy, dummy, dummy, (784, 32, 32, 10), 60000, 10000, 1)
        for k, v in kw.items():
            setattr(b, k, v)
        return b

    def rej(b, nd=500, match="", p=plan):
        rc = L.mbd_mnist_step_launch(ctypes.byref(p), nd, ctypes.byref(b), None)
        assert rc == -1 and match in L.mbd_last_error().decode(), L.mbd_last_error().decode()

    rej(bufs(layers=(784, 64, 32, 10)), match="784-32-32-10")
    rej(bufs(), nd=1, match="Ndiffuse")
    rej(bufs(keys_dev=None), match="keys")
    rej(bufs(test_images_dev=None), match="test set")
    rej(bufs(n_train=100), match="N must lie")
    rej(bufs(eval_every=0), match="eval_every")
    p2 = _lib.StepPlan.from_buffer_copy(plan)
    p2.n_total = p2.n_local = 0
    rej(bufs(), match="N must lie", p=p2)
    p3 = _lib.StepPlan.from_buffer_copy(plan)
    p3.nu = 100
    rej(bufs(), match="nu = 26506", p=p3)
    p4 = _lib.StepPlan.from_buffer_copy(plan)
    p4.weights_dev = None
    rej(bufs(), match="plan buffer", p=p4)
    assert L.mbd_mnist_forward(None, 1, ctypes.byref(bufs()), None, 1, None, None, None) == -1
