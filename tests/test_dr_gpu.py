"""Domain randomisation of the vector env on the device (DESIGN.md §5n): the drawn factor table and every output held bit for bit to
the specification (dr_factors, and a second VecEnv whose table the host sets), [1, 1] ranges equal to the nominal env, batch and
permutation invariance across both kernel mappings, graph replay, the refusals of a real plan, the trainers, and run_mpc's policy row."""
import ctypes

import numpy as np
import pytest
import torch

from mbd_b200 import _lib, prng
from mbd_b200.envs import get_env
from mbd_b200.envs.vec import VecEnv, dr_factors, env_spec
from mbd_b200.rl import networks as nets
from mbd_b200.rl import ppo, sac
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu

FR, GR = (0.5, 1.5), (0.7, 1.3)
_cache = {}


def _env(name):
    if name not in _cache:
        _cache[name] = get_env(name)
    return _cache[name]


def _actions(env, steps, n, seed):
    return torch.as_tensor(np.random.default_rng(seed).uniform(-1, 1, (steps, n, env.action_size)).astype(np.float32), device="cuda")


def _outputs(s):
    return [x.detach().cpu().numpy().reshape(s.obs.shape[0], -1).copy() for x in (s.raw, s.reward, s.obs, s.done, s.truncation)]


def _same(a, b, what, rows_a=slice(None), rows_b=slice(None)):
    for name, u, v in zip(("raw", "reward", "obs", "done", "truncation"), a, b):
        assert_bit_exact(u[rows_a], v[rows_b], f"{what}: {name}")


def _spec_table(dkeys, episodes, fr=FR, gr=GR):
    return np.float32([dr_factors(k, int(e), fr, gr) for k, e in zip(dkeys, episodes)])


def _table(venv):
    return venv.factors.cpu().numpy()


@pytest.mark.parametrize("name", ["hopper", "humanoidrun"])
def test_matches_the_specification(name):
    """the table after every step is dr_factors of each env's episode, and every output equals a VecEnv whose table the host sets
    to those factors before each step"""
    env, B, T, ep = _env(name), 33, 30, 5
    dkeys, rkeys = ppo.dr_keys(4, B), prng.split(prng.PRNGKey(5), B)
    acts = _actions(env, T, B, seed=6)
    venv = VecEnv(env, B, ep)
    venv.set_domain_randomization(FR, GR, dkeys)
    ref = VecEnv(env, B, ep)
    ref.set_model_factors(friction=np.ones(B), gear=np.ones(B))
    _same(_outputs(venv.reset(rkeys)), _outputs(ref.reset(rkeys)), f"{name} reset")
    e = np.zeros(B, np.int64)
    resets = 0
    for t in range(T):
        spec = _spec_table(dkeys, e)
        assert_bit_exact(_table(venv), spec, f"{name} table before step {t}")
        assert np.array_equal(venv.dr_episodes.cpu().numpy(), e)
        ref.set_model_factors(friction=spec[:, 0], gear=spec[:, 1])
        got, want = _outputs(venv.step(acts[t])), _outputs(ref.step(acts[t]))
        _same(got, want, f"{name} step {t}")
        done = got[3].reshape(-1) != 0
        e += done
        resets += int(done.sum())
    assert resets >= B * (T // ep - 1)
    assert len(np.unique(_table(venv)[:, 0])) == B   # every env its own draw


@pytest.mark.parametrize("name", ["hopper", "humanoidrun"])
def test_unit_ranges_equal_the_nominal_env(name):
    env, B, T, ep = _env(name), 33, 30, 5
    rkeys = prng.split(prng.PRNGKey(7), B)
    acts = _actions(env, T, B, seed=8)
    venv, nom = VecEnv(env, B, ep), VecEnv(env, B, ep)
    venv.set_domain_randomization((1, 1), (1, 1), ppo.dr_keys(0, B))
    _same(_outputs(venv.reset(rkeys)), _outputs(nom.reset(rkeys)), f"{name} reset")
    for t in range(T):
        _same(_outputs(venv.step(acts[t])), _outputs(nom.step(acts[t])), f"{name} step {t}")
    assert (venv.factors == 1).all() and int(venv.dr_episodes.min()) == T // ep


def _run(env, dkeys, rkeys, acts, ep=5):
    venv = VecEnv(env, len(dkeys), ep)
    venv.set_domain_randomization(FR, GR, dkeys)
    venv.reset(rkeys)
    out = []
    for t in range(acts.shape[0]):
        out.append(_outputs(venv.step(acts[t])) + [_table(venv).copy()])
    return out


@pytest.mark.parametrize("name", ["hopper", "humanoidrun"])
def test_batch_and_permutation_invariance(name):
    """env b's factors and trajectory depend on its keys and actions only: B = 1, 33 and 4096 (the 11-link humanoid crosses from the
    lane-per-link to the warp-per-link kernel) and a permutation of 33 envs"""
    env, N, T = _env(name), 4096, 20
    dkeys, rkeys = ppo.dr_keys(2, N), prng.split(prng.PRNGKey(3), N)
    acts = _actions(env, T, N, seed=4)
    full = _run(env, dkeys, rkeys, acts)
    for B in (1, 33):
        part = _run(env, dkeys[:B], rkeys[:B], acts[:, :B].contiguous())
        for t in range(T):
            for k, (u, v) in enumerate(zip(part[t], full[t])):
                assert_bit_exact(u, v[:B], f"{name} B = {B} step {t} output {k}")
    perm = np.random.default_rng(0).permutation(33)
    pt = _run(env, dkeys[perm], rkeys[perm], acts[:, torch.as_tensor(perm, device="cuda")].contiguous())
    for t in range(T):
        for k, (u, v) in enumerate(zip(pt[t], full[t])):
            assert_bit_exact(u, v[perm], f"{name} permuted step {t} output {k}")


def test_graph_replay_equals_eager():
    env, B, T = _env("hopper"), 64, 20
    dkeys, rkeys = ppo.dr_keys(1, B), prng.split(prng.PRNGKey(1), B)
    acts = _actions(env, T, B, seed=1)
    eager = _run(env, dkeys, rkeys, acts, ep=4)
    venv = VecEnv(env, B, 4)
    venv.set_domain_randomization(FR, GR, dkeys)
    venv.reset(rkeys)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        venv.step()
    for t in range(T):
        venv.actions.copy_(acts[t])
        g.replay()
        got = _outputs(venv._view()) + [_table(venv).copy()]
        for k, (u, v) in enumerate(zip(got, eager[t])):
            assert_bit_exact(u, v, f"graph step {t} output {k}")
    assert int(venv.dr_episodes.min()) == T // 4


BAD = [dict(range=(np.nan, 1, 1, 1)), dict(range=(1, np.inf, 1, 1)), dict(range=(-1, 1, 1, 1)), dict(range=(1, 1, 1.3, 0.7)),
       dict(keys_dev=None), dict(episodes_dev=None), dict(factors_dev=None)]


@pytest.mark.parametrize("bad", BAD, ids=[next(iter(b)) + str(i) for i, b in enumerate(BAD)])
def test_refusals_leave_the_device_untouched(bad):
    env, B = _env("hopper"), 8
    venv = VecEnv(env, B, 5)
    venv.set_domain_randomization(FR, GR, ppo.dr_keys(0, B))
    venv.reset(prng.split(prng.PRNGKey(0), B))
    torch.cuda.synchronize()
    before = [t.clone() for t in (venv.state, venv.obs, venv.factors, venv.dr_episodes, venv.steps)]
    P = _lib.VecPlan.from_buffer_copy(venv.plan)
    D = _lib.VecDr.from_buffer_copy(venv.dr)
    for k, v in bad.items():
        if k == "range":
            D.range[:] = [float(x) for x in v]
        elif k == "factors_dev":
            P.factors_dev = v
        else:
            setattr(D, k, v)
    L = _lib.lib()
    keys = prng.split(prng.PRNGKey(1), B)
    kt = torch.as_tensor(keys.view(np.int32), device="cuda")
    for rc in (L.mbd_vec_step_dr(ctypes.byref(P), ctypes.byref(D), None),
               L.mbd_vec_reset_dr(ctypes.byref(P), ctypes.byref(D), ctypes.c_void_p(kt.data_ptr()), None)):
        assert rc == -1
    torch.cuda.synchronize()
    for a, b in zip(before, (venv.state, venv.obs, venv.factors, venv.dr_episodes, venv.steps)):
        assert torch.equal(a, b)
    for name in ("car2d", "pushT"):
        flat = VecEnv(_env(name), B)
        assert L.mbd_vec_step_dr(ctypes.byref(flat.plan), ctypes.byref(venv.dr), None) == -1
        assert "xpbd envs only" in L.mbd_last_error().decode()


def test_set_model_factors_ends_randomization():
    env, B = _env("hopper"), 4
    venv = VecEnv(env, B, 5)
    venv.set_domain_randomization(FR, GR, ppo.dr_keys(0, B))
    assert venv.dr.keys_dev == venv.dr_keys.data_ptr() and venv.dr.episodes_dev == venv.dr_episodes.data_ptr()
    assert venv.plan.factors_dev == venv.factors.data_ptr()
    venv.set_model_factors(gear=0.8)
    assert venv.dr is None and (venv.factors[:, 1] == np.float32(0.8)).all()
    venv.set_model_factors()
    assert not venv.plan.factors_dev and venv.dr is None


# ---- the trainers -------------------------------------------------------------------------------------------------------------
PPO_CFG = dict(num_timesteps=128, episode_length=7, num_envs=8, num_eval_envs=16, batch_size=4, num_minibatches=4, unroll_length=4,
               num_updates_per_batch=2, num_evals=2, normalize_observations=True, learning_rate=3e-4, seed=3)
SAC_CFG = dict(num_timesteps=16 + 3 * 8, episode_length=5, num_envs=8, num_eval_envs=16, batch_size=16, grad_updates_per_step=4,
               min_replay_size=16, max_replay_size=64, num_evals=2, normalize_observations=True, reward_scaling=30.0, seed=1)


def _bits(a, b, what):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), what


@pytest.mark.parametrize("algo", ["ppo", "sac"])
def test_unit_randomization_trains_as_nominal(algo):
    train, env, cfg = (ppo.train, "halfcheetah", PPO_CFG) if algo == "ppo" else (sac.train, "hopper", SAC_CFG)
    _, nom, m0 = train(_env(env), **cfg)
    _, dr, m1 = train(_env(env), randomization=dict(friction_range=(1, 1), gear_range=(1.0, 1.0)), **cfg)
    assert nom.keys() == dr.keys()
    for k in nom:
        _bits(nom[k], dr[k], f"{algo}: {k}")
    assert m0["eval/episode_reward"] == m1["eval/episode_reward"]


@pytest.mark.parametrize("algo", ["ppo", "sac"])
def test_training_envs_draw_and_evaluation_stays_nominal(algo):
    dr = dict(friction_range=FR, gear_range=GR)
    if algo == "ppo":
        tr = ppo.PPOTrainer(_env("halfcheetah"), 128, 7, 8, 16, 3e-4, 1e-3, 0.97, 3, 4, 4, 4, 2, 2, True, 1.0, 0.3, 0.95,
                            randomization=dr)
    else:
        tr = sac.SACTrainer(_env("hopper"), 80, 5, 8, 16, 6e-4, 0.997, 1, 16, 2, True, 30.0, 0.005, 16, 64, 4, randomization=dr)
    assert np.array_equal(tr.dr_keys, ppo.dr_keys(3 if algo == "ppo" else 1, 8))
    first = _table(tr.venv).copy()
    assert_bit_exact(first, _spec_table(tr.dr_keys, np.zeros(8)), "episode 0")
    tr.capture()
    if algo == "sac":
        tr.prefill()           # 2 env steps, then 4 more: one auto-reset at step 5
    for _ in range(2 if algo == "ppo" else 4):
        tr.training_step()
    tr.evaluate()
    torch.cuda.synchronize()
    e = tr.venv.dr_episodes.cpu().numpy()
    table = _table(tr.venv)
    assert (e >= 1).all()
    assert_bit_exact(table, _spec_table(tr.dr_keys, e), "the table after training")
    assert (table[:, 0] >= np.float32(FR[0])).all() and (table[:, 0] <= np.float32(FR[1])).all()
    assert (table[:, 1] >= np.float32(GR[0])).all() and (table[:, 1] <= np.float32(GR[1])).all()
    assert not np.array_equal(table, first)
    assert not tr.evenv.plan.factors_dev and tr.evenv.dr is None and tr.evenv.factors is None


# ---- the policy row ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo", ["ppo", "sac"])
def test_policy_row_equals_a_written_loop(algo):
    from mbd_b200.scripts import run_mpc
    env, Nstep, seeds = _env("hopper"), 12, (0, 3, 5)
    O, nu = env_spec(env).obs_size, env.action_size
    sizes = nets.policy_sizes(O, nu) if algo == "ppo" else nets.sac_policy_sizes(O, nu)
    rng = np.random.default_rng(0)
    params = dict(policy=nets.init_params(prng.PRNGKey(11), sizes), mean=rng.normal(0, 0.1, O).astype(np.float32),
                  std=rng.uniform(0.5, 2, O).astype(np.float32))
    states0 = run_mpc.initial_states(env, seeds)
    Actor = ppo.Actor if algo == "ppo" else sac.Actor
    for fr, gr in ((1.0, 1.0), (0.5, 0.7), (1.5, 1.3)):
        got = run_mpc.policy_rewards(env, algo, params, states0, seeds, Nstep, fr, gr)
        want = []
        for i, s in enumerate(seeds):
            venv = VecEnv(env, 1)
            if (fr, gr) != (1.0, 1.0):
                venv.set_model_factors(friction=fr, gear=gr)
            venv.set_state(states0[i:i + 1])
            act = Actor(venv, *(torch.as_tensor(params[k]).cuda() for k in ("policy", "mean", "std")))
            keys = prng.split(prng.PRNGKey((3 << 32) | s), Nstep)
            r = []
            for c in range(Nstep):
                act.act(keys[c])
                r.append(float(venv.step().reward[0]))
            want.append(np.mean(np.float64(np.float32(r))))
        assert np.array_equal(got, np.float64(want)), (fr, gr, got, want)
