"""The fused SAC update without a GPU: include/mbd_sac_learn.h's host harness (g++ -ffp-contract=off, the kernel's association
orders) against the float64 contract of tests/sac_learn_ref.py on the families of tests/sac_learn_families.py, Adam and Polyak
against float64, the deliberate mistakes of an fp32 mirror, the ABI's refusals, and the learner options."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from mbd_b200.rl import networks as nets
from tests import sac_learn_families as fam
from tests import sac_learn_ref as ref
from tests import sac_ref
from tests.rl_ref import ratio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_f32p = ctypes.POINTER(ctypes.c_float)
f32 = np.float32


def _fp(a):
    return a.ctypes.data_as(_f32p)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sac_learn") / "libsac_learn_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "host_sac_learn", "sac_learn_harness.cpp"), "-o", so], check=True,
                   env={**os.environ, "CC": "", "CXX": ""})
    L = ctypes.CDLL(so)
    L.sac_learn_update_host.argtypes = [_f32p] * 9 + [ctypes.c_longlong] + [_f32p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_float] * 4 \
        + [_f32p] * 4
    L.sac_adam_host.argtypes = [_f32p] * 4 + [ctypes.c_int, ctypes.c_float, ctypes.c_longlong]
    L.sac_polyak_host.argtypes = [_f32p, _f32p, ctypes.c_int, ctypes.c_float]
    return L


def host_update(L, f, lr=6e-4, tau=0.005, step=0, moments=None):
    """one update of the harness on family f: dict of the new state, the fp32 gradients and the losses"""
    O, nu, n = f["O"], f["nu"], f["rows"].shape[0]
    c = lambda a: np.array(a, f32, copy=True)   # noqa: E731
    s = dict(policy=c(f["policy"]), q=c(f["q"]), target_q=c(f["target_q"]), log_alpha=c(f["log_alpha"]))
    mo = moments or {}
    s.update(pm=c(mo.get("pm", np.zeros_like(s["policy"]))), pv=c(mo.get("pv", np.zeros_like(s["policy"]))),
             qm=c(mo.get("qm", np.zeros_like(s["q"]))), qv=c(mo.get("qv", np.zeros_like(s["q"]))), amv=c(mo.get("amv", np.zeros(2))))
    out = dict(gp=np.zeros_like(s["policy"]), gq=np.zeros_like(s["q"]), ga=np.zeros(1, f32), losses=np.zeros(3, f32))
    L.sac_learn_update_host(*[_fp(s[k]) for k in ("policy", "q", "target_q", "log_alpha", "pm", "pv", "qm", "qv", "amv")], step,
                            *[_fp(c(f[k])) for k in ("mean", "std", "rows", "eps")], O, nu, n, lr, f["reward_scaling"],
                            f["discounting"], tau, _fp(out["gp"]), _fp(out["gq"]), _fp(out["ga"]), _fp(out["losses"]))
    s.update(out)
    return s


def grad_ratios(f, gp, gq, ga) -> dict:
    C = ref.contract(f["policy"], f["q"], f["target_q"], f["log_alpha"], f["mean"], f["std"], f["rows"], f["eps"], f["O"], f["nu"],
                     f["reward_scaling"], f["discounting"])
    return {k: float(ratio(g, C[k]).max()) for k, g in (("policy", gp), ("q", gq), ("alpha", ga))}, C


def test_contract_values_are_brax_gradients():
    """the contract's float64 values of the formulas equal torch autograd in float64 (sac_ref.grads64) on a hopper-sized family.
    The contract takes discounting and reward_scaling as the fp32 words the kernel reads, grads64 as Python floats: 1e-7 relative"""
    f = fam.base(11, 3, 64, 0)
    _, C = grad_ratios(f, f["policy"], f["q"], f["log_alpha"])
    ls, ga, gq, gp = sac_ref.grads64(f["policy"], f["q"], f["target_q"], f["log_alpha"], f["mean"], f["std"], f["rows"], f["eps"],
                                     f["O"], f["nu"], f["reward_scaling"], f["discounting"])
    for got, want in ((C["policy"].v, gp), (C["q"].v, gq), (C["alpha"].v, ga)):
        assert np.abs(got - want).max() <= 1e-7 * max(np.abs(want).max(), 1e-30)
    assert np.allclose(C["losses"].v, ls, rtol=1e-7, atol=1e-12)


@pytest.mark.parametrize("O,nu,n", [s for s in fam.MILD if s[2] < 512 or (s[0], s[1]) in ((11, 3), (128, 32), (1, 1))])
def test_harness_mild_shapes(harness, O, nu, n):
    f = fam.base(O, nu, n, O * 100 + nu)
    s = host_update(harness, f)
    r, C = grad_ratios(f, s["gp"], s["gq"], s["ga"])
    assert max(r.values()) <= ref.K, r
    assert float(ratio(s["losses"], C["losses"]).max()) <= ref.K


@pytest.mark.parametrize("name", sorted(fam.families().keys()))
def test_harness_families(harness, name):
    f = fam.families()[name]
    s = host_update(harness, f)
    r, C = grad_ratios(f, s["gp"], s["gq"], s["ga"])
    assert max(r.values()) <= ref.K, r
    if name == "all_truncated":
        assert not s["gq"].any()          # no row reaches Q: its gradient is exactly zero


def test_adam_subnormal_v(harness):
    """second moments in the subnormal range and gradients whose square is subnormal, against float64 Adam"""
    rng = np.random.default_rng(3)
    n = 4096
    p = rng.standard_normal(n).astype(f32)
    g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, -17, n)).astype(f32)
    m = (rng.standard_normal(n) * 1e-25).astype(f32)
    v = (rng.random(n) * 1e-39).astype(f32)
    assert (v < np.finfo(f32).tiny).all()
    want_p, _, want_v = ref.adam(p, m, v, g, 6e-4, 5000)
    pp, mm, vv = p.copy(), m.copy(), v.copy()
    harness.sac_adam_host(_fp(pp), _fp(mm), _fp(vv), _fp(g), n, 6e-4, 5000)
    assert np.isfinite(pp).all()
    assert float(ratio(pp, want_p).max()) <= ref.K


@pytest.mark.parametrize("t", [1, 7, 1_000_003])
def test_adam_polyak(harness, t):
    """Adam at step 1, at a step with non-zero moments and at a step count past 10^6, and Polyak, against float64 given the
    harness's own fp32 gradient"""
    rng = np.random.default_rng(t)
    n = 4096
    p = rng.standard_normal(n).astype(f32)
    g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 1, n)).astype(f32)
    m = np.zeros(n, f32) if t == 1 else (rng.standard_normal(n) * 1e-3).astype(f32)
    v = np.zeros(n, f32) if t == 1 else (rng.random(n) * 1e-5).astype(f32)
    want_p, want_m, want_v = ref.adam(p, m, v, g, 6e-4, t)
    pp, mm, vv = p.copy(), m.copy(), v.copy()
    harness.sac_adam_host(_fp(pp), _fp(mm), _fp(vv), _fp(g), n, 6e-4, t)
    for got, want in ((pp, want_p), (mm, want_m), (vv, want_v)):
        assert float(ratio(got, want).max()) <= ref.K
    tgt = rng.standard_normal(n).astype(f32)
    out = tgt.copy()
    harness.sac_polyak_host(_fp(out), _fp(pp), n, 0.005)
    assert float(ratio(out, ref.polyak(tgt, pp, 0.005)).max()) <= ref.K


# ---- an fp32 mirror and its deliberate mistakes ---------------------------------------------------------------------------------------
def mirror(f, mistake=None, lr=6e-4, tau=0.005):
    """one sgd_step in torch fp32 (autograd) and numpy fp32 Adam, with an optional deliberate mistake: (gp, gq, ga, new state)"""
    O, nu = f["O"], f["nu"]
    t = lambda a, g=False: torch.tensor(np.asarray(a, f32), requires_grad=g)   # noqa: E731
    pol, q, la = t(f["policy"], True), t(f["q"], True), t(f["log_alpha"], True)
    tq, mean, std, rows, eps = t(f["target_q"]), t(f["mean"]), t(f["std"]), t(f["rows"]), t(f["eps"])
    psizes, qsizes = nets.sac_policy_sizes(O, nu), nets.sac_q_sizes(O, nu)
    obs, action, reward, discount, next_obs, trunc = (rows[:, :O], rows[:, O:O + nu], rows[:, O + nu], rows[:, O + nu + 1],
                                                      rows[:, O + nu + 2:2 * O + nu + 2], rows[:, 2 * O + nu + 2])
    x, xn = (obs - mean) / std, (next_obs - mean) / std
    logits = nets.relu_mlp(x, nets.unflatten(pol, psizes))
    loc, s = logits.chunk(2, -1)
    scale = torch.nn.functional.softplus(s) + nets.MIN_STD
    lp_a = nets.log_prob(logits, eps[0] * scale + loc)
    alpha_loss = torch.mean(torch.exp(la) * (-lp_a + 0.5 * nu).detach())
    ga = torch.autograd.grad(alpha_loss, la)[0]
    la_new = la.detach() - ALPHA_STEP(ga)
    alpha = torch.exp(la_new if mistake == "new_alpha_in_critic" else la).detach()
    through = mistake == "grad_through_target"
    pn = pol if through else pol.detach()
    ln = nets.relu_mlp(xn, nets.unflatten(pn, psizes))
    locn, sn = ln.chunk(2, -1)
    raw_c = eps[1] * (torch.nn.functional.softplus(sn) + nets.MIN_STD) + locn
    red = (lambda a: torch.max(a, 0).values) if mistake == "max_not_min" else (lambda a: torch.min(a, 0).values)
    next_v = red(nets.sac_q(nets.sac_q_unflatten(tq, qsizes), xn, torch.tanh(raw_c))) - alpha * nets.log_prob(ln, raw_c)
    target = reward * f["reward_scaling"] + discount * f["discounting"] * next_v
    if not through:
        target = target.detach()
    qv = nets.sac_q(nets.sac_q_unflatten(q, qsizes), x, action)
    mask = 1.0 if mistake == "no_trunc_mask" else (1.0 - trunc)
    err = (qv - target) * mask
    critic_loss = 0.5 * (torch.sum(err * err) / err.shape[1] if mistake == "critic_mean_over_n" else torch.mean(err * err))
    gq, gp_c = torch.autograd.grad(critic_loss, [q, pol], allow_unused=True)
    qn_np = adam_np(f["q"], gq.numpy(), lr, mistake)
    qa_src = torch.tensor(qn_np) if mistake == "new_q_in_actor" else q.detach()
    raw_p = eps[2] * scale + loc
    qa = nets.sac_q(nets.sac_q_unflatten(qa_src, qsizes), x, torch.tanh(raw_p))
    actor_loss = torch.mean(torch.exp(la).detach() * nets.log_prob(logits, raw_p) - red(qa))
    gp = torch.autograd.grad(actor_loss, pol)[0]
    if gp_c is not None:
        gp = gp + gp_c
    pn_np = adam_np(f["policy"], gp.numpy(), lr, mistake)
    tq_np = np.asarray(f["target_q"], f32)
    toward = np.asarray(f["q"], f32) if mistake == "polyak_to_old_q" else qn_np
    tq_new = (tq_np + f32(tau) * (toward - tq_np)).astype(f32)
    return gp.numpy(), gq.numpy(), ga.numpy(), dict(policy=pn_np, q=qn_np, target_q=tq_new)


def ALPHA_STEP(ga):
    return ref.ALPHA_LR * torch.sign(ga)


def adam_np(p, g, lr, mistake):
    """torch's Adam at step 1 from zero moments, fp32"""
    g = np.asarray(g, f32)
    m = (f32(0.1) * g).astype(f32)
    v = (f32(0.001) * (g * g)).astype(f32)
    bc1, bc2 = (f32(1.0), f32(1.0)) if mistake == "no_bias_correction" else (f32(1 - 0.9), f32(1 - 0.999))
    return (np.asarray(p, f32) - f32(lr) / bc1 * (m / (np.sqrt(v) / np.sqrt(bc2) + f32(1e-8)))).astype(f32)


MISTAKES = ["critic_mean_over_n", "new_q_in_actor", "new_alpha_in_critic", "polyak_to_old_q", "no_trunc_mask", "no_bias_correction",
            "grad_through_target", "max_not_min"]


def mirror_ratio(f, mistake):
    """the largest distance in radii of the mirror's gradients and of its new parameters (Adam and Polyak given the correct
    mirror's gradient) from the contract"""
    gp, gq, ga, st = mirror(f, mistake)
    r, _ = grad_ratios(f, gp, gq, ga)
    _, gq0, _, st0 = mirror(f, None)
    gp0 = mirror(f, None)[0]
    z = lambda a: np.zeros_like(np.asarray(a, f32))   # noqa: E731
    wp = ref.adam(f["policy"], z(f["policy"]), z(f["policy"]), gp0, 6e-4, 1)[0]
    wq = ref.adam(f["q"], z(f["q"]), z(f["q"]), gq0, 6e-4, 1)[0]
    r["policy_new"] = float(ratio(st["policy"], wp).max())
    r["q_new"] = float(ratio(st["q"], wq).max())
    r["target_new"] = float(ratio(st["target_q"], ref.polyak(f["target_q"], st0["q"], 0.005)).max())
    return max(r.values()), r


def _mistake_family():
    f = fam.base(11, 3, 64, 11, reward_scaling=30.0, discounting=0.997)
    f["log_alpha"][:] = f32(0.5)
    return f


def test_mirror_meets_the_bound():
    worst, r = mirror_ratio(_mistake_family(), None)
    assert worst <= ref.K, r


@pytest.mark.parametrize("mistake", MISTAKES)
def test_mistakes_leave_the_bound(mistake):
    worst, r = mirror_ratio(_mistake_family(), mistake)
    print(f"{mistake}: {worst:.3g} radii")
    assert worst > 10 * ref.K, r


# ---- ABI, refusals, options -----------------------------------------------------------------------------------------------------------
def test_scratch_size_matches_harness(harness):
    from mbd_b200 import ops
    out = ctypes.c_longlong()
    harness.sac_learn_scratch_host.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong)]
    for O, nu, n in ((11, 3, 512), (128, 32, 4096), (1, 1, 1)):
        harness.sac_learn_scratch_host(O, nu, n, ctypes.byref(out))
        assert ops.sac_learn_scratch(O, nu, n) == out.value


def _plan():
    from mbd_b200 import _lib
    P = _lib.SacLearnPlan()
    P.O, P.nu, P.batch, P.updates = 11, 3, 512, 64
    for name, _ in P._fields_:
        if name.endswith("_dev"):
            setattr(P, name, 0x1000)          # never dereferenced: every refusal comes before any CUDA call
    P.scratch_floats = 1 << 40
    return P


@pytest.mark.parametrize("field,value", [("O", 0), ("O", 129), ("nu", 0), ("nu", 33), ("batch", 0), ("batch", 4097), ("updates", 0),
                                         ("scratch_floats", 10), ("policy_dev", 0), ("q_dev", 0), ("target_q_dev", 0),
                                         ("log_alpha_dev", 0), ("policy_m_dev", 0), ("policy_v_dev", 0), ("q_m_dev", 0),
                                         ("q_v_dev", 0), ("alpha_mv_dev", 0), ("std_dev", 0),
                                         ("ctl_dev", 0), ("mean_dev", 0), ("batch_dev", 0), ("eps_dev", 0), ("upd_ctl_dev", 0),
                                         ("scratch_dev", 0), ("losses_dev", 0)])
def test_refusals_before_cuda(field, value):
    from mbd_b200 import _lib
    P = _plan()
    setattr(P, field, value)
    L = _lib.lib()
    assert L.mbd_sac_update(ctypes.byref(P), None) != 0
    assert b"mbd_sac_update" in L.mbd_last_error()
    assert L.mbd_sac_update(None, None) != 0


def test_learner_option_parsing():
    import inspect

    from mbd_b200.rl import sac, train_sac
    assert inspect.signature(sac.train).parameters["learner"].default == "torch"
    assert inspect.signature(sac.SACTrainer).parameters["learner"].default == "torch"
    with pytest.raises(ValueError, match="learner"):
        sac.train("hopper", 100000, 1000, learner="jax")
    with pytest.raises(SystemExit):
        train_sac.main(["--learner", "jax"])
    seen = {}

    def fake_train(**kw):
        seen.update(kw)
        raise RuntimeError("stop")
    orig = sac.train
    sac.train = fake_train
    try:
        for argv, want in (([], "torch"), (["--learner", "fused"], "fused")):
            with pytest.raises(RuntimeError, match="stop"):
                train_sac.main(argv + ["--num_timesteps", "9000"])
            assert seen["learner"] == want
    finally:
        sac.train = orig
