"""pushT's loop on the device against float64, substep by substep over a whole horizon (tests/pusht_chain.py), without the oracle.

tests/test_pusht_f64_gpu.py holds one physics step of `k_pusht`.  This file holds the loop around it on the starts, control
sequences, mu and solver modes of tests/test_pusht_horizon_ref_cpu.py (the scripted push is generated closed loop on the kernel
here; the kernel and the oracle agree bit for bit, so it is the same sequence):
* `k_pusht` at n = 1, 77, 129 and at one n of several CTAs per SM with a ragged last CTA (row b replays sequence b mod 2): the
  NSUB = 1 launch with repeated controls is the NSUB = 5 launch bit for bit, rows that replay one sequence are bit-identical,
  and every substep of the checked rows is within K radii of pusht_ref.step of the kernel's own state before it;
* the recurrent state is the 16 words q | qd: a relaunch (H = 1) from the state after env step t - 1 gives env step t bit for
  bit, and with NSUB = k its k-th substep;
* the production solve within the measured truncation constant, and the sweep-cap and undecided fractions within the caps of
  the CPU file;
* `k_pusht_ps` (the vector env, MPC plant) stepped 50 times from per-env starts equals `k_pusht`'s trajectory and rewards bit
  for bit, and the fused sampling path (`pusht_rollout(key=...)`) equals `k_pusht` on the controls it drew, so the checks
  above cover both."""
import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops
from mbd_b200.envs.vec import VecEnv
from tests import horizon_ref as HR
from tests import pusht_chain as C
from tests import pusht_ref as X
from tests.test_pusht_horizon_ref_cpu import K, MODES, MUS, NOT_FIXED_CAP, SWEEP_CAP, UNDECIDED_CAP
from tests.test_pusht_ref_cpu import table

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NS = (1, 77, 129)
RELAUNCH_STEPS = (0, 1, 25, 49)
WORST = {}                  # (n, start, mu, mode) -> largest ratio, printed at the end


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def big_n():
    """several 64-thread CTAs per SM and a ragged last CTA"""
    return 4 * 64 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def _rows(n):
    """the rows of a large launch held to float64: the first 129, every 41st and the last 40 (the ragged last CTA)"""
    return np.unique(np.r_[0:129, 129:n:41, n - 40:n])


def kernel(P, st, Y, **kw):
    o = ops.pusht_rollout(T(P), T(st), T(Y), **kw)
    return {k: v.cpu().numpy() for k, v in o.items() if v is not None}


def kernel_step(P):
    return lambda s, u: kernel(P, s, np.reshape(u, (1, 1, 2)), want_final=True)["final"][0]


def relaunch(P, prev, u):
    one = kernel_step(P)
    return np.stack([one(s, a) for s, a in zip(prev, u)])


@pytest.fixture(scope="module")
def memo():
    return C.StepMemo()


@pytest.fixture(scope="module")
def starts():
    """[(label, state, Y [2, H, 2])]: the starts of pusht_chain with the scripted push (closed loop on k_pusht) and the random
    sequence of the CPU file"""
    env = mbd_b200.envs.get_env("pushT")
    return [(label, st, C.sequences(kernel_step(env.params), env.params, st, off, 300 + si))
            for si, (label, st, off) in enumerate(C.starts(env))]


@pytest.mark.parametrize("n", NS + ("big",))
def test_k_pusht_chain_within_the_bound(memo, starts, n):
    n = big_n() if n == "big" else n
    seq = np.arange(n) % 2
    rows = _rows(n) if n > 129 else np.arange(n)
    for label, st, Y2 in starts:
        Y = Y2[seq]
        U = C.substep_controls(Y)
        for mu in MUS:
            for mode in MODES:
                P1 = X.solver_params(table(mu), mode, nsub=1)
                P5 = X.solver_params(table(mu), mode, nsub=C.NSUB)
                one = kernel(P1, st, U, want_traj=True, want_final=True)
                five = kernel(P5, st, Y, want_traj=True, want_final=True, want_rewss=True)
                traj = one["traj"]
                what = f"n={n} {label} mu={mu} {mode}"
                assert HR.same_bits(traj[:, C.NSUB - 1::C.NSUB], five["traj"]), f"{what}: NSUB = 1 and NSUB = 5 trajectories"
                assert HR.same_bits(one["final"], five["final"]), f"{what}: NSUB = 1 and NSUB = 5 final states"
                for j in range(min(n, 2)):     # one thread per sample, nothing shared: equal controls give equal words
                    assert HR.same_bits(traj[seq == j], np.broadcast_to(traj[j], traj[seq == j].shape)), f"{what}: rows of sequence {j}"
                prev = C.previous(st, traj[rows]).reshape(-1, 16)
                got, u = traj[rows].reshape(-1, 16), U[rows].reshape(-1, 2)
                res = C.check(memo, P1, mode, prev, got, u)
                WORST[(n, label, mu, mode)] = res["ratio"]
                assert res["ratio"] <= K, f"{what}: {res['ratio']:.3g} radii"
                assert res["finite"], what
                assert res["undecided"].mean() <= UNDECIDED_CAP[label], what
                if n != NS[1]:
                    continue
                # at n = 77: the solver along both sequences, and the relaunches of the last row
                two = slice(0, 2 * C.NSUB * C.H)
                prev2, got2, u2 = prev[two], got[two], u[two]
                if mode == "prod":
                    ref2 = {key: v[two] for key, v in res["ref"].items()}
                    tr = C.truncation_ratio(got2, relaunch(X.solver_params(table(mu), "fixed", nsub=1), prev2, u2), ref2)
                    WORST[("truncation", label, mu, mode)] = tr
                    assert tr <= X.TRUNC_MEASURED, f"{what}: truncation ratio {tr:.4g}"
                    capped = (relaunch(X.solver_params(table(mu), "prod", nsub=1, iters=200), prev2, u2) != got2).any(1)
                    assert capped.mean() <= SWEEP_CAP[label], f"{what}: {capped.mean():.3f} of the substeps at the sweep cap"
                else:
                    nf = (relaunch(X.solver_params(table(mu), "fixed", nsub=1, iters=8000), prev2, u2) != got2).any(1)
                    assert nf.mean() <= NOT_FIXED_CAP[label], f"{what}: {nf.mean():.3f} of the substeps not at a fixed point"
                b = n - 1
                prev5 = HR.previous_states(st, five["traj"])
                for t in RELAUNCH_STEPS:
                    o = kernel(P5, prev5[b, t], Y[b:b + 1, t:t + 1], want_final=True, want_rewss=True)
                    assert HR.same_bits(o["final"][0], five["traj"][b, t]), f"{what}: relaunch of env step {t}"
                    assert HR.same_bits(o["rewss"][0], five["rewss"][b, t:t + 1]), f"{what}: reward of env step {t}"
                    for ks in range(1, C.NSUB + 1):
                        o = kernel(X.solver_params(table(mu), mode, nsub=ks), prev5[b, t], Y[b:b + 1, t:t + 1], want_final=True)
                        assert HR.same_bits(o["final"][0], traj[b, C.NSUB * t + ks - 1]), f"{what}: env step {t} with NSUB = {ks}"


def test_k_pusht_ps_equals_k_pusht_over_the_horizon(starts):
    """the vector env (shipped table) from per-env starts, stepped H times: every state and reward equal k_pusht's (NSUB = 5) from
    that start bit for bit; no env is done, so none is reset"""
    env = mbd_b200.envs.get_env("pushT")
    S = len(starts)
    nenv = 4 * S + 5
    which, seq = np.arange(nenv) % S, (np.arange(nenv) // S) % 2
    venv = VecEnv(env, nenv, episode_length=C.H + 10)
    venv.set_state(np.stack([starts[j][1] for j in which]))
    Y = np.stack([starts[j][2][s] for j, s in zip(which, seq)])
    raw, rew = [], []
    for t in range(C.H):
        out = venv.step(T(Y[:, t]))
        assert not out.done.any().item(), f"an env is done at step {t}"
        raw.append(out.raw.cpu().numpy().copy())
        rew.append(out.reward.cpu().numpy().copy())
    raw, rew = np.stack(raw, 1), np.stack(rew, 1)
    for j, (label, st, _) in enumerate(starts):
        idx = np.flatnonzero(which == j)
        o = kernel(env.params, st, Y[idx], want_traj=True, want_rewss=True)
        assert HR.same_bits(raw[idx], o["traj"]), f"{label}: states"
        assert HR.same_bits(rew[idx], o["rewss"]), f"{label}: rewards"


def test_fused_sampling_equals_k_pusht_on_its_draws(starts):
    """pusht_rollout(key=...) with n_begin > 0 and a ragged n: its returns equal k_pusht on the controls it wrote, bit for bit"""
    env = mbd_b200.envs.get_env("pushT")
    st = starts[3][1]
    for H_ in (1, C.H):
        n_total, n_begin, n_local = 4096, 1029, 77
        Ybar = T((np.random.default_rng(H_).normal(size=(H_, 2)) * 0.3).astype(np.float32))
        Y0s = torch.empty((n_local, H_, 2), device=DEV)
        o = ops.pusht_rollout(T(env.params), T(st), Y0s, want_rewss=True, key=np.uint32([3, H_]), n_total=n_total,
                              n_begin=n_begin, sigma=0.7, Ybar=Ybar)
        Y = Y0s.cpu().numpy()
        assert (np.abs(Y) == 1).any() and (np.abs(Y) <= 1).all()
        ref = kernel(env.params, st, Y, want_rewss=True)
        assert HR.same_bits(o["rews"].cpu().numpy(), ref["rews"]), f"H={H_}: rews"
        assert HR.same_bits(o["rewss"].cpu().numpy(), ref["rewss"]), f"H={H_}: rewss"


def test_report(memo):
    """the largest |kernel - f64| / radius per (n, start, mu, mode) and the truncation ratios over the tests above"""
    for k in sorted(WORST, key=str):
        print(k, round(WORST[k], 3))
    print("float64 substep evaluations:", memo.evaluated)
