"""Every CUDA rollout kernel's loop against the float64 horizon reference (tests/horizon_ref.py), without the oracle.

tests/test_xpbd_f64_gpu.py holds one substep (H = 1, nsub_override = 1) and one reward of each kernel.  This file holds the
loop around them on the same (model, variant) cases, at n = 1, 77 and 129, and at one n above 16 x SMs where the
selector picks the kernel itself:
* the substep chain, k = 1 .. n_frames, on every family state, each substep teacher-forced on the kernel's own state;
* the env-step chain at H = 50 (and 60 for humanoidtrack) from the reset pose and one state per family: prefix runs equal
  to the full run bit for bit, every reward, the tracked positions, the return and the demo log-density;
* that the loop carries nothing but the 13 words per link: a relaunch from a substep's or an env step's state (n = 1)
  gives the next one bit for bit, and the relaunched substeps along the horizon stay within the bound;
* the fused sampling kernels, whose returns equal `ops.rollout` on the actions they drew, so the checks above cover them;
* the vector env's per-env-state kernels (`k_rollout<PerEnv>`, `k_rollout_wpl<PerEnv>`, `k_pusht_ps`): one family state per env,
  next state and reward bit for bit against the broadcast kernel from that state, reward within the float64 bound."""
import hashlib

import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import ops
from mbd_b200.envs.vec import VecEnv
from mbd_b200.model import blob as B
from tests import horizon_ref as HR
from tests import pusht_families as PF
from tests import pusht_ref as PX
from tests import xpbd_families as F
from tests.test_horizon_ref_cpu import HORIZON_MODELS, HORIZON_UNDECIDED, chain_undecided_cap, horizon_actions, horizon_starts, starts
from tests.test_xpbd_f64_gpu import CASES, HUMANOIDS, launched_kernel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 2.0
NS = (1, 77, 129)
H = 50
RELAUNCH_STEPS = (0, 1, 25, 49)      # env steps of the last finite sample relaunched substep by substep
# undecided fraction of those relaunched substeps where one H100 run measured more than the CPU file's per-model cap (few
# substeps per case; at n = 1 the relaunched sample is the bang-bang one): measured fraction beside each cap
RELAUNCH_UNDECIDED = {"humanoidrun": 0.065,        # 12 of 196 (n = 1)
                      "ant": 0.025,                # 5 of 240 (n = 129)
                      "halfcheetah": 0.012,        # 5 of 448 (n = 129)
                      "contact_params": 0.008}     # 1 of 140
# fraction of the random-action samples (all but the saturated sample 0) that may blow up to inf / NaN over the horizon:
# 1 of 2148 measured (humanoidstandup from the reset pose at n = 2149; the CPU oracle blows up on it at the same step 44)
BLOWUP = 0.001
WORST = {}                           # (kernel, family) -> largest ratio, printed at the end


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def big_n():
    return 16 * sms() + 37


def ps_kernel(blob, nenv):
    """the kernel `mbd_vec_step` (csrc/mbd_b200.cu) runs for an xpbd vector env of nenv envs"""
    return "k_rollout<PerEnv>" if int(blob.view(np.int32)[B.H_NLINK]) == 11 and nenv <= 16 * sms() else "k_rollout_wpl<PerEnv>"


VEC_CASES = [(m, 67) for m in F.SHIPPED + ["contact_params", "gen3"]] + [(m, "big") for m in HUMANOIDS + ["gen100"]]


def test_every_kernel_is_covered(tmp_path):
    """the cases below launch every rollout kernel after the launcher's remapping, and every per-env-state kernel"""
    got = {launched_kernel(F.make_env(m, tmp_path).blob, v, n, sms()) for m, v in CASES for n in NS}
    got |= {launched_kernel(F.make_env(m, tmp_path).blob, 0, big_n(), sms()) for m in HUMANOIDS}
    got |= {ps_kernel(F.make_env(m, tmp_path).blob, big_n() if nb == "big" else nb) for m, nb in VEC_CASES}
    got.add("k_pusht_ps")      # test_vecenv_pusht_step_within_the_float64_bound: the only kernel of the pushT vector env
    want = {"lane-per-link", "wpl-cta", "wpl-named", "wpl-generic", "pk-group", "k_rollout<PerEnv>", "k_rollout_wpl<PerEnv>", "k_pusht_ps"}
    assert want <= got, want - got


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def kernel_run(m, ntrack):
    def run(st, Y, nsub=0, xref=None):
        o = ops.rollout(m, T(st), T(Y), xref=None if xref is None else T(xref), want_rewss=True, want_final=True,
                        want_track=ntrack > 0, nsub_override=nsub)
        return {k: (None if v is None else v.cpu().numpy()) for k, v in o.items()}
    return run


@pytest.fixture(scope="module")
def memo():
    return HR.StepMemo()


_HORIZON_MEMO = {}


def check_horizon_memo(blob, st, Y, full, traj, xref):
    """HR.check_horizon, shared by the launches that hand it the same words (it is a function of its inputs only)"""
    h = hashlib.sha1()
    for a in (blob, st, Y, traj, xref) + tuple(full[k] for k in sorted(full) if full[k] is not None):
        if a is not None:
            h.update(np.ascontiguousarray(a).tobytes())
    key = h.hexdigest()
    if key not in _HORIZON_MEMO:
        _HORIZON_MEMO[key] = HR.check_horizon(blob, st, Y, full, traj, xref)
    return _HORIZON_MEMO[key]


def _note(kernel, fam, q):
    WORST[(kernel, fam)] = max(WORST.get((kernel, fam), 0.0), q)


def _rows(n):
    """the samples of an n above 16 x SMs whose substeps are checked: the first 129 (shared with the smaller n), every 41st
    and the last 40 (the ragged last CTA)"""
    return np.unique(np.r_[0:129, 129:n:41, n - 40:n])


def _cases_with_n(models=None):
    out = [(m, v, n) for m, v in CASES for n in NS if models is None or m in models]
    return out + [(m, 0, "big") for m in HUMANOIDS]


@pytest.mark.parametrize("name,variant,n", _cases_with_n())
def test_substep_chain_within_the_bound(tmp_path, memo, name, variant, n):
    env = F.make_env(name, tmp_path)
    n = big_n() if n == "big" else n
    m = env.device_model(torch.device(DEV))
    kern = launched_kernel(env.blob, variant, n, sms())
    run = kernel_run(m, 0)
    nsub = int(env.blob.view(np.int32)[3])
    ops.set_kernel_variant(variant)
    try:
        fams = F.FAMILIES if n <= 129 else ["F1", "F5"]
        for fam in fams:
            und = tot = 0
            for i, (st, u) in enumerate(F.build(env, fam, max(n, 8))):
                u = u[:n]
                ch = HR.substep_chain(run, st, u, nsub)
                rows = _rows(n) if n > 129 else np.arange(n)
                prev = np.concatenate([c[rows] for c in ch[:-1]])
                got = np.concatenate([c[rows] for c in ch[1:]])
                q, nu_ = HR.step_ratio(memo, env.blob, prev, np.tile(u[rows], (nsub, 1)), got)
                _note(kern, fam, q)
                assert q <= K, f"{name} v{variant} n={n} {fam}[{i}]: substep chain {q:.3g} radii"
                und, tot = und + nu_, tot + len(prev)
                if i == 0:      # the recurrent state is the 13 words per link: relaunch the last sample one substep at a time
                    b = n - 1
                    for k in range(1, nsub + 1):
                        one = run(ch[k - 1][b], u[b:b + 1, None], nsub=1)["final"][0]
                        assert HR.same_bits(one, ch[k][b]), f"{name} v{variant} n={n} {fam}: relaunch of substep {k}"
            if n > 1 and tot:
                assert und <= chain_undecided_cap(name, fam) * tot, f"{name} {fam}: {und} of {tot} substeps undecided"
    finally:
        ops.set_kernel_variant(0)


@pytest.mark.parametrize("name,variant,n", _cases_with_n(HORIZON_MODELS))
def test_env_step_chain_within_the_bound(tmp_path, memo, name, variant, n):
    env = F.make_env(name, tmp_path)
    n = big_n() if n == "big" else n
    m = env.device_model(torch.device(DEV))
    kern = launched_kernel(env.blob, variant, n, sms())
    blob = env.blob
    ntrack = int(blob.view(np.int32)[B.H_NTRACK])
    run = kernel_run(m, ntrack)
    nsub = int(blob.view(np.int32)[3])
    xref = env.xref if name == "humanoidtrack" else None
    ops.set_kernel_variant(variant)
    try:
        sts = horizon_starts(env, name, run, xref)
        sts = sts if n <= 129 else sts[:2]
        und = tot = 0
        for si, (label, st, xref) in enumerate(sts):
            for H_ in ((H, 60) if xref is not None else (H,)):
                Y = horizon_actions(env.action_size, n, H_, 1000 + si)
                full, traj = HR.env_step_chain(run, st, Y, xref)
                for k, q in check_horizon_memo(blob, st, Y, full, traj, xref).items():
                    _note(kern, f"{label} {k}", q)
                    assert q <= K, f"{name} v{variant} n={n} {label} H={H_} {k}: {q:.3g} radii"
                # one env step relaunched from the loop's own state, then the same step one substep at a time
                ok = HR.finite_samples(traj)
                assert (~ok[1:]).sum() <= BLOWUP * n, f"{name} v{variant} n={n} {label}: samples {np.flatnonzero(~ok)} blew up"
                prev = HR.previous_states(st, traj)
                b = int(np.flatnonzero(ok)[-1]) if ok.any() else -1
                for t in (RELAUNCH_STEPS if b >= 0 else ()):
                    one = run(prev[b, t], Y[b:b + 1, t:t + 1])["final"][0]
                    assert HR.same_bits(one, traj[b, t]), f"{name} v{variant} n={n} {label}: relaunch of env step {t}"
                    ch = HR.relaunch_chain(run, prev[b, t], Y[b, t], nsub)
                    assert HR.same_bits(ch[-1], traj[b, t]), f"{name} v{variant} n={n} {label}: substeps of env step {t}"
                    q, nu_ = HR.step_ratio(memo, blob, np.stack(ch[:-1]), np.tile(Y[b, t], (nsub, 1)), np.stack(ch[1:]))
                    _note(kern, f"{label} relaunch", q)
                    assert q <= K, f"{name} v{variant} n={n} {label}: relaunched substeps of step {t}: {q:.3g} radii"
                    und, tot = und + nu_, tot + nsub
        cap = max(HORIZON_UNDECIDED[name], RELAUNCH_UNDECIDED.get(name, 0.0))
        assert und <= cap * tot, f"{name}: {und} of {tot} relaunched substeps undecided"
    finally:
        ops.set_kernel_variant(0)


@pytest.mark.parametrize("variant", [0, 1, 2, 3, 8])
@pytest.mark.parametrize("name", ["humanoidrun", "humanoidtrack"])
def test_fused_sampling_equals_rollout_of_its_draws(name, variant):
    """ops.sample_rollout with a ragged n_local and n_begin > 0: its returns (and logpd) equal ops.rollout on the actions it
    wrote to Y0s bit for bit, so every check above covers the fused kernels too"""
    env = mbd_b200.envs.get_env(name)
    m = env.device_model(torch.device(DEV))
    st = F.build(env, "F1", 8)[0][0]
    nu = env.action_size
    xref = T(env.xref) if name == "humanoidtrack" else None
    ops.set_kernel_variant(variant)
    try:
        for H_ in (1, 50):
            n_total, n_begin, n_local = 4096, 1029, 77
            Ybar = T((np.random.default_rng(H_).normal(size=H_ * nu) * 0.3).astype(np.float32))
            Y0s = torch.empty((n_local, H_ * nu), device=DEV)
            rews = torch.empty(n_local, device=DEV)
            lp = torch.empty(n_local, device=DEV) if xref is not None else None
            ops.sample_rollout(m, T(st), np.uint32([3, H_]), n_total, n_begin, n_local, H_, 0.7, Ybar, Y0s, rews, xref=xref,
                               logpd_out=lp)
            Y = Y0s.view(n_local, H_, nu).contiguous()
            assert (Y.abs() == 1).any() and (Y.abs() <= 1).all()
            ref = ops.rollout(m, T(st), Y, xref=xref)
            assert HR.same_bits(rews.cpu().numpy(), ref["rews"].cpu().numpy()), f"{name} v{variant} H={H_}: rews"
            if lp is not None:
                assert HR.same_bits(lp.cpu().numpy(), ref["logpd"].cpu().numpy()), f"{name} v{variant} H={H_}: logpd"
    finally:
        ops.set_kernel_variant(0)


def _family_states(env, name):
    out = [st for _, st in starts(env, name)]
    for fam in F.FAMILIES:
        out += [st for st, _ in F.build(env, fam, 8)[1:]]
    return out


@pytest.mark.parametrize("name,nenv", VEC_CASES)
def test_vecenv_step_within_the_float64_bound(tmp_path, name, nenv):
    """k_rollout<PerEnv> / k_rollout_wpl<PerEnv>: env b starts at family state b mod S with its own action.  Its next state and reward
    equal ops.rollout from that state bit for bit; its reward is within the float64 bound of its own two states."""
    env = F.make_env(name, tmp_path)
    nenv = big_n() if nenv == "big" else nenv
    blob = env.blob
    S = _family_states(env, name)
    which = np.arange(nenv) % len(S)
    U = F.actions(env.action_size, nenv, 17)
    s0 = np.stack([S[j] for j in which])
    venv = VecEnv(env, nenv)
    venv.set_state(s0.reshape(nenv, -1))
    out = venv.step(T(U))
    raw, rew = out.raw.cpu().numpy().copy(), out.reward.cpu().numpy().copy()
    m = env.device_model(torch.device(DEV))
    for j in range(len(S)):
        idx = np.flatnonzero(which == j)
        o = ops.rollout(m, T(S[j]), T(U[idx][:, None]), want_final=True)
        assert HR.same_bits(raw[idx], o["final"].cpu().numpy()), f"{name} B={nenv} state {j}: next state"
        assert HR.same_bits(rew[idx], o["rews"].cpu().numpy()), f"{name} B={nenv} state {j}: reward"
    r = HR.step_rewards(blob, s0, raw[:, None], U[:, None])
    q = HR.ratio(rew, r.v[:, 0], r.r[:, 0])
    _note(ps_kernel(blob, nenv), f"{name} reward", q)
    assert q <= K, f"{name} B={nenv}: reward {q:.3g} radii"


def test_vecenv_pusht_step_within_the_float64_bound():
    """k_pusht_ps: every pushT family state in one ragged batch; next state and reward bit for bit against ops.pusht_rollout
    from each state, the reward within the float64 bound of the env's own next state"""
    env = mbd_b200.envs.get_env("pushT")
    params = env.device_params()
    S = [st for fam in PF.FAMILIES for st, _ in PF.build(fam, 8)]
    nenv = len(S) + 67
    which = np.arange(nenv) % len(S)
    U = PF.controls(nenv, 23)
    venv = VecEnv(env, nenv)
    venv.set_state(np.stack([S[j] for j in which]))
    out = venv.step(T(U))
    raw, rew = out.raw.cpu().numpy().copy(), out.reward.cpu().numpy().copy()
    for j in range(len(S)):
        idx = np.flatnonzero(which == j)
        o = ops.pusht_rollout(params, T(S[j]), T(U[idx][:, None]), want_final=True)
        assert HR.same_bits(raw[idx], o["final"].cpu().numpy()), f"pushT state {j}: next state"
        assert HR.same_bits(rew[idx], o["rews"].cpu().numpy()), f"pushT state {j}: reward"
    r = PX.reward(raw)
    q = HR.ratio(rew, r.v, r.r)
    _note("k_pusht_ps", "reward", q)
    assert q <= K, f"pushT reward: {q:.3g} radii"


def test_pusht_rewards_over_the_horizon():
    """k_pusht at H = 50 from family states: every step's reward against the float64 reward of that step's trajectory state,
    and the return against sum(rewss) / H"""
    env = mbd_b200.envs.get_env("pushT")
    params = env.device_params()
    for fam in ("free", "box0", "both", "limits_both", "theta"):
        for i, (st, u) in enumerate(PF.build(fam, 77)[:2]):
            Y = np.clip(np.random.default_rng(i).normal(size=(77, H, 2)) * 0.8, -1.0, 1.0).astype(np.float32)
            Y[:, 0] = u
            o = ops.pusht_rollout(params, T(st), T(Y), want_traj=True, want_rewss=True)
            traj, rewss, rews = (o[k].cpu().numpy() for k in ("traj", "rewss", "rews"))
            ref = PX.reward(traj)
            q = HR.ratio(rewss, ref.v, ref.r)
            ret = HR.mean_return(rewss)
            q2 = HR.ratio(rews, ret.v, ret.r)
            _note("k_pusht", f"{fam} horizon", max(q, q2))
            assert q <= K and q2 <= K, f"{fam}[{i}]: rewards {q:.3g}, return {q2:.3g} radii"


def test_report():
    """the largest |kernel - f64| / radius per (kernel, family) over the tests above"""
    for k in sorted(WORST):
        print(f"{k[0]:18s} {k[1]:24s} {WORST[k]:.3f}")
