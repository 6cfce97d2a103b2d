"""Black-box solves on the device (mbd_bbo_batch_step_launch): launch (1) against the oracles bit for bit and against the float64
objective bound, the MPPI tail against its float64 contract, batches against B = 1 bit for bit, graph replay against eager
launches, the past-the-end guard, a staged solve against the host restatement at every step, and the reference's defaults."""
import numpy as np
import pytest
import torch

from mbd_b200 import ops
from mbd_b200.blackbox import mbd_opt
from mbd_b200.planners.engine import make_schedule
from tests import bbo_oracle as bo
from tests import bbo_ref as br
from tests import tail_ref as tr

pytestmark = pytest.mark.gpu
f32 = np.float32


def N_(t):
    return t.detach().cpu().numpy()


def _engine(fn, dim, N, seeds, Nd=100, temp=1.0):
    e = mbd_opt.BboEngine(fn, dim, N, [temp] * len(seeds), Nd)
    sig = make_schedule(1e-4, 1e-2, Nd)[3]
    pk = [mbd_opt.problem_keys(s, Nd) for s in seeds]
    e.load_schedule([k for k, _ in pk], sig, [k0 for _, k0 in pk])
    e.set_step(Nd - 1)
    return e, sig, pk


def _check_step(orc, e, b, fn, t, sig, pk, mu, temp, what):
    """step t of problem b just ran with mean mu (None: the first step's per-sample draw): Y0s, J and best_hist bit for bit,
    J within the float64 bound, Ybars[t - 1] within the MPPI tail's float64 contract"""
    x_min, x_max = br.DOMAINS[fn]
    keys, k0 = pk[b]
    Y = N_(e.Y0s[b])
    want = br.sample(orc, keys[t], float(sig[t]), mu, k0, e.N, e.HNu)
    assert np.array_equal(Y.view(np.uint32), want.view(np.uint32)), what + ": Y0s"
    J = N_(e.rews[b])
    assert np.array_equal(J.view(np.uint32), bo.bbo_eval(fn, Y, x_min, x_max).view(np.uint32)), what + ": J vs oracle"
    assert N_(e.best_hist[b, t]).view(np.uint32) == J.max().view(np.uint32), what + ": best_hist"
    J64, rad = br.reference(fn, Y, x_min, x_max)
    br.check_J(J, J64, rad, what + ": J vs float64")
    ref = tr.reference(J, temp, Y0s=Y)
    sc = N_(e.scalars[b])
    depth = tr.cluster_depth(e.N)
    tr.check_stats(ref, J, sc[0], sc[1], depth, what)
    wb = tr.weight_bounds(ref, depth, sc[0], sc[1])
    tr.check_weights(ref, N_(e.weights[b]), wb, what + ": weights")
    nruns = (e.N + ops.RUN - 1) // ops.RUN
    tr.check_columns(N_(e.Ybars[b, t - 1]), ref["Ybar"], tr.ybar_bound(ref, Y, wb["rho"], tr.wsum_depth(nruns)), what + ": mean")


@pytest.mark.parametrize("N", [1, 7, 64, 65, 2048])
@pytest.mark.parametrize("dim", [1, 2, 255, 256, 257, 800, 6912])
@pytest.mark.parametrize("fn", ["Ackley", "Rastrigin", "Levy"])
def test_first_and_later_step(orc, fn, dim, N):
    Nd, temp = 100, 1.0
    e, sig, pk = _engine(fn, dim, N, [3], Nd, temp)
    e.step()
    torch.cuda.synchronize()
    _check_step(orc, e, 0, fn, Nd - 1, sig, pk, None, temp, f"{fn} dim={dim} N={N} first step")
    mu = N_(e.Ybars[0, Nd - 2])
    e.step()
    torch.cuda.synchronize()
    _check_step(orc, e, 0, fn, Nd - 2, sig, pk, mu, temp, f"{fn} dim={dim} N={N} second step")
    assert int(e.ctl[0, 0].item()) == Nd - 3
    assert np.isneginf(N_(e.best_hist[0, :Nd - 2])).all(), "only the steps that ran write best_hist"


def _solve(fn, dim, N, seeds, Nd, graph):
    e, _, _ = _engine(fn, dim, N, seeds, Nd)
    if graph:
        e.capture()
    for _ in range(Nd - 1):
        e.step()
    torch.cuda.synchronize()
    e.check_exchange()
    return e


def _outputs(e):
    return dict(Ybars=N_(e.Ybars), rew_hist=N_(e.rew_hist), best_hist=N_(e.best_hist), Y0s=N_(e.Y0s), rews=N_(e.rews))


@pytest.mark.parametrize("fn,seeds", [("Rastrigin", [0, 1, 2, 3, 4, 5]), ("Ackley", [5, 3, 0, 4, 2, 1]),
                                      ("Levy", [16, 3, 9, 0, 12, 5, 1, 14, 7, 2, 11, 4, 15, 8, 6, 13, 10])])
def test_batch_matches_single_problems(fn, seeds):
    """every problem of a batch (B = 6, or 17; permuted seed orders) reproduces its B = 1 solve bit for bit"""
    dim, N, Nd = 800, 64, 100
    out = _outputs(_solve(fn, dim, N, seeds, Nd, graph=True))
    for b, s in enumerate(seeds):
        solo = _outputs(_solve(fn, dim, N, [s], Nd, graph=False))
        for k in ("Ybars", "rew_hist", "best_hist", "Y0s", "rews"):
            assert np.array_equal(out[k][b].view(np.uint32), solo[k][0].view(np.uint32)), f"{fn} seed {s} (b={b}): {k}"


@pytest.mark.parametrize("fn", ["Ackley", "Rastrigin", "Levy"])
def test_graph_replay_matches_eager_and_stops_at_the_end(fn):
    seeds, dim, N, Nd = [0, 1, 2], 257, 65, 20
    eg = _solve(fn, dim, N, seeds, Nd, graph=True)
    ea = _solve(fn, dim, N, seeds, Nd, graph=False)
    og, oa = _outputs(eg), _outputs(ea)
    for k in og:
        assert np.array_equal(og[k].view(np.uint32), oa[k].view(np.uint32)), f"{fn}: {k} graph vs eager"
    assert (N_(eg.ctl[:, 0]) == 0).all()
    eg.step()   # one replay past step 1: the counter is at 0, so nothing may be written
    torch.cuda.synchronize()
    after = _outputs(eg)
    for k in og:
        assert np.array_equal(after[k].view(np.uint32), og[k].view(np.uint32)), f"{fn}: replay past the end wrote {k}"
    with pytest.raises(ops.MbdError, match="ran past step 1"):
        eg.check_exchange()


@pytest.mark.parametrize("fn", ["Ackley", "Rastrigin", "Levy"])
def test_device_step_vs_host_step(orc, fn):
    """at every step of a solve the device's mu_t is staged into the host restatement: draws and J bit for bit, the next mean
    within the tail's float64 contract"""
    dim, N, Nd, temp = 800, 64, 100, 1.0
    e, sig, pk = _engine(fn, dim, N, [0, 7], Nd, temp)
    e.capture()
    for t in range(Nd - 1, 0, -1):
        mus = [None if t == Nd - 1 else N_(e.Ybars[b, t]) for b in range(2)]
        e.step()
        torch.cuda.synchronize()
        for b in range(2):
            _check_step(orc, e, b, fn, t, sig, pk, mus[b], temp, f"{fn} b={b} step {t}")


@pytest.mark.parametrize("fn", ["Rastrigin", "Ackley", "Levy"])
def test_reference_defaults_improve(orc, fn, capsys):
    """at mbd_opt.py's defaults (6 seeds x 64 samples x 800 dims, 100 steps) the mean over seeds of Js.max() ends above where it
    starts, on the device and in the host restatement at the same seeds (both curves are printed)"""
    a = mbd_opt.Args(fn_name=fn)
    xs, ys, mus = mbd_opt.run_exp_batch(a, list(range(a.Nexp)))
    assert xs.tolist() == [64 * k for k in range(1, 100)] and ys.shape == (6, 99) and mus.shape == (6, 800)
    xs1, ys1 = mbd_opt.run_exp(a, 2)
    assert np.array_equal(ys1.view(np.uint32), ys[2].view(np.uint32)), "run_exp is the batch of one"
    sig = make_schedule(a.beta0, a.betaT, a.Ndiffuse)[3]
    host = []
    for s in range(a.Nexp):
        keys, k0 = mbd_opt.problem_keys(s, a.Ndiffuse)
        host.append(br.host_solve(orc, bo.bbo_eval, fn, s, a.Nsample, a.dim, a.Ndiffuse, a.temp_sample, sig, keys, k0)[0])
    dev, hst = ys.mean(axis=0), np.mean(host, axis=0)
    with capsys.disabled():
        pick = [0, 9, 19, 39, 59, 79, 98]
        print(f"\n[bbo] {fn}-800d mean Js.max() at steps {[k + 1 for k in pick]}: device {np.round(dev[pick], 2).tolist()} "
              f"host {np.round(hst[pick], 2).tolist()}")
    assert dev[-1] > dev[0], f"{fn}: device curve {dev[0]} -> {dev[-1]}"
    assert hst[-1] > hst[0], f"{fn}: host curve {hst[0]} -> {hst[-1]}"
