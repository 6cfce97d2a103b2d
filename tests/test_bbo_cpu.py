"""Black-box solves without a device: mbd_bbo_batch_step_launch refuses bad arguments before any CUDA call (with a message), Args
carries mbd_opt.py's constants, the key chain is mbd_opt.py's, and the saved curve has the reference's shape."""
import ctypes

import numpy as np
import pytest

from mbd_b200 import _lib, prng
from mbd_b200.blackbox import mbd_opt

FAKE = 0x1000   # never dereferenced: every case below fails validation, which runs before the first CUDA call


def _plan(**kw):
    """a black-box plan (H = 1, nu = dim, no model) that passes every check except the one a test breaks"""
    p = _lib.StepPlan()
    for f in ("params_dev", "ctl_dev", "Ybars_dev", "Y0s_dev", "rews_dev", "rews_all_dev", "logp_dev", "weights_dev", "runs_dev",
              "partial_dev", "scalars_dev"):
        setattr(p, f, FAKE)
    p.n_total, p.n_begin, p.n_local, p.H, p.nu, p.P, p.rank, p.temp = 64, 0, 64, 1, 800, 1, 0, 1.0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _bufs(**kw):
    b = _lib.BboBufs(FAKE, FAKE, -5.0, 5.0)
    for k, v in kw.items():
        setattr(b, k, v)
    return b


def _reject(p, B=6, Nd=100, fn=2, bufs=None):
    L = _lib.lib()
    rc = L.mbd_bbo_batch_step_launch(ctypes.byref(p) if p is not None else None, B, Nd, fn, None,
                                     ctypes.byref(bufs) if bufs is not None else None, None)
    return rc, L.mbd_last_error().decode()


@pytest.mark.parametrize("kw,B,Nd,fn,bufs,msg", [
    ({}, 6, 100, 0, {}, "unknown fn"),
    ({}, 6, 100, 4, {}, "unknown fn"),
    ({"H": 2, "nu": 400}, 6, 100, 2, {}, "H must be 1"),
    ({"model": FAKE}, 6, 100, 2, {}, "no model and no demonstration"),
    ({"xref_dev": FAKE, "href": 5, "logpd_dev": FAKE, "logpd_all_dev": FAKE}, 6, 100, 1, {}, "no model and no demonstration"),
    ({"nu": 27 * 256 + 1}, 6, 100, 3, {}, "H * Nu exceeds 27 * 256 columns"),
    ({"n_total": 1 << 20, "n_local": 1 << 20, "nu": 4096}, 1, 100, 2, {}, "below 2^32"),
    ({}, 6, 100, 2, {"init_keys_dev": None}, "init_keys and best_hist must be set"),
    ({}, 6, 100, 2, {"best_hist_dev": None}, "init_keys and best_hist must be set"),
    ({}, 6, 100, 2, {"x_min": 5.0, "x_max": 5.0}, "x_min < x_max"),
    ({}, 6, 100, 2, {"x_min": 5.0, "x_max": -5.0}, "x_min < x_max"),
    ({}, 6, 100, 2, {"x_min": float("nan")}, "x_min < x_max"),
    ({}, 0, 100, 2, {}, "B must be at least 1"),
    ({}, 65536, 100, 2, {}, "B must be at most 65535"),
    ({}, 6, 1, 2, {}, "Ndiffuse must be at least 2"),
    ({"P": 2, "peer_base_ptrs": ctypes.cast(FAKE, ctypes.POINTER(ctypes.c_uint64))}, 6, 100, 2, {}, "P must be 1"),
    ({"weights_dev": None}, 6, 100, 1, {}, "a work buffer is NULL"),
    ({"n_local": 32}, 6, 100, 1, {}, "n_local == n_total"),
], ids=["fn0", "fn4", "H2", "model", "xref", "columns", "counter-2^32", "init-keys", "best-hist", "empty-domain", "reversed-domain",
        "nan-domain", "B0", "B65536", "Nd1", "P2", "weights", "nlocal"])
def test_bbo_launch_rejects_with_message(kw, B, Nd, fn, bufs, msg):
    rc, err = _reject(_plan(**kw), B, Nd, fn, _bufs(**bufs))
    assert rc == -1, (rc, err)
    assert err.startswith("mbd_bbo_batch_step_launch: ") and msg in err, err


def test_bbo_launch_null_plan_and_bufs_rejected():
    assert _reject(None)[0] == -1 and "plan is NULL" in _reject(None, bufs=_bufs())[1]
    rc, err = _reject(_plan(), bufs=None)
    assert rc == -1 and "bufs is NULL" in err, err


def test_args_defaults_are_the_reference_constants():
    a = mbd_opt.Args()
    assert (a.fn_name, a.dim, a.Nexp, a.Nsample, a.Ndiffuse, a.temp_sample, a.beta0, a.betaT) == \
        ("Rastrigin", 800, 6, 64, 100, 1.0, 1e-4, 1e-2)
    assert mbd_opt.DOMAINS == {"Ackley": (-5.0, 10.0), "Rastrigin": (-5.0, 5.0), "Levy": (-5.0, 5.0)}
    assert set(mbd_opt.DOMAINS) == set(_lib.BBO_FNS)


@pytest.mark.parametrize("seed", [0, 5, 123456789])
def test_key_chain_and_first_step_key(seed):
    """rng = PRNGKey(seed); every step `rng, Y0s_rng = split(rng)` (no reset split, no rng_exp split; the warm-up call does
    not advance it); the first step's mean is drawn with PRNGKey(seed) itself"""
    Nd = 100
    keys, k0 = mbd_opt.problem_keys(seed, Nd)
    assert k0.tolist() == prng.PRNGKey(seed).tolist()
    rng = prng.PRNGKey(seed)
    for t in range(Nd - 1, 0, -1):
        rng, sub = prng.split(rng)
        assert keys[t].tolist() == sub.tolist(), t
    assert keys[0].tolist() == [0, 0]


def test_output_file_shape(tmp_path):
    a = mbd_opt.Args()
    xs = mbd_opt.sample_counts(a)
    assert xs.tolist() == [64 * k for k in range(1, 100)]
    ys = np.linspace(-9000.0, -2000.0, 99)
    path = str(tmp_path / "bbo" / "Rastrigin-800d_MBD.npy")
    mbd_opt.write_result(xs, ys, path)
    out = np.load(path)
    assert out.shape == (2, 99) and out.dtype == np.float32
    assert out[0].tolist() == [64.0 * k for k in range(1, 100)]
    assert np.array_equal(out[1], ys.astype(np.float32))
    assert mbd_opt.result_path(a).endswith("results/bbo/Rastrigin-800d_MBD.npy")


def test_batch_args_checked_before_the_device(monkeypatch):
    with pytest.raises(KeyError):
        mbd_opt.check_batch_args(mbd_opt.Args(fn_name="Sphere"), [0])
    with pytest.raises(ValueError, match="at least one seed"):
        mbd_opt.check_batch_args(mbd_opt.Args(), [])
    with pytest.raises(ValueError, match="Ndiffuse must be at least 2"):
        mbd_opt.check_batch_args(mbd_opt.Args(Ndiffuse=1), [0])
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        mbd_opt.run_exp_batch(mbd_opt.Args(), [0, 1])
