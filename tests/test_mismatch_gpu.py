"""Model factors of the vector env on the device (DESIGN.md §5k): an all-ones table steps exactly as no table, env b steps exactly as
a nominal VecEnv of its specification scaled_env(env, F[b]) under both kernel mappings, envs permute with their factor rows, a
captured step follows in-place rewrites of the table, and the receding-horizon controllers run against per-problem plants."""
import numpy as np
import pytest
import torch

from mbd_b200 import prng
from mbd_b200.envs import get_env
from mbd_b200.envs.vec import VecEnv, scaled_env
from mbd_b200.planners import mbd_mpc, pi_mpc
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu

XPBD = ["humanoidrun", "humanoidstandup", "humanoidtrack", "hopper", "walker2d", "cartpole", "ant", "halfcheetah"]
COMBOS = [(f, g) for f in (0.0, 0.3, 1.7) for g in (0.5, 1.4)]
T = 30
_cache = {}


def _env(name):
    if name not in _cache:
        _cache[name] = get_env(name)
    return _cache[name]


def _actions(env, steps, n, seed):
    return torch.as_tensor(np.random.default_rng(seed).uniform(-1, 1, (steps, n, env.action_size)).astype(np.float32), device="cuda")


def _trajectory(venv, acts):
    """[steps] of (raw, reward, obs, done) on the host"""
    out = []
    for t in range(acts.shape[0]):
        s = venv.step(acts[t])
        out.append([x.detach().cpu().numpy().reshape(venv.num_envs, -1) for x in (s.raw, s.reward, s.obs, s.done)])
    return out


def _same(a, b, what, rows_a=slice(None), rows_b=slice(None)):
    for t, (xa, xb) in enumerate(zip(a, b)):
        for name, u, v in zip(("raw", "reward", "obs", "done"), xa, xb):
            assert_bit_exact(u[rows_a], v[rows_b], f"{what}: {name}, step {t}")


@pytest.mark.parametrize("name", XPBD)
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_all_ones_equals_no_table(name, n):
    """for the 11-link models, 33 envs run the lane-per-link kernel and 4096 the warp-per-link one"""
    env = _env(name)
    keys = prng.split(prng.PRNGKey(1), n)
    acts = _actions(env, T, n, seed=2)
    nominal = VecEnv(env, n)
    nominal.reset(keys)
    ones = VecEnv(env, n)
    ones.set_model_factors(friction=1.0, gear=1.0)
    assert ones.plan.factors_dev == ones.factors.data_ptr() and (ones.factors == 1).all()
    ones.reset(keys)
    _same(_trajectory(nominal, acts), _trajectory(ones, acts), f"{name}, B = {n}")


@pytest.mark.parametrize("name,n", [("hopper", 12), ("ant", 12), ("walker2d", 12), ("halfcheetah", 12), ("cartpole", 12),
                                    ("humanoidrun", 12), ("humanoidrun", 4096), ("humanoidstandup", 12), ("humanoidstandup", 4096)])
def test_env_b_equals_its_specification(name, n):
    """env b with factors F[b] (friction in {0, 0.3, 1.7}, gear in {0.5, 1.4}) = a nominal VecEnv of scaled_env(env, F[b]), bit for
    bit; and it differs from the nominal env, so the factors are not ignored"""
    env = _env(name)
    F = np.float32([COMBOS[b % len(COMBOS)] for b in range(n)])
    keys = prng.split(prng.PRNGKey(3), n)
    acts = _actions(env, T, n, seed=4)
    venv = VecEnv(env, n)
    venv.set_model_factors(friction=F[:, 0], gear=F[:, 1])
    venv.reset(keys)
    got = _trajectory(venv, acts)
    nominal = VecEnv(env, n)
    nominal.reset(keys)
    nom = _trajectory(nominal, acts)
    for k, (f, g) in enumerate(COMBOS):
        rows = np.flatnonzero(np.arange(n) % len(COMBOS) == k)
        spec = VecEnv(scaled_env(env, f, g), len(rows))
        spec.reset(keys[rows])
        _same(got, _trajectory(spec, acts[:, torch.as_tensor(rows, device="cuda")]), f"{name}, F = ({f}, {g})", rows_a=rows)
        for b in rows:
            assert any((x[0][b] != y[0][b]).any() for x, y in zip(got, nom)), f"env {b} (F = ({f}, {g})) equals the nominal env"


@pytest.mark.parametrize("name", ["hopper", "humanoidrun"])
def test_permuting_envs_with_their_factors_permutes_the_outputs(name):
    env, n = _env(name), 12
    rng = np.random.default_rng(5)
    F = rng.uniform(0.0, 2.0, (n, 2)).astype(np.float32)
    keys = prng.split(prng.PRNGKey(6), n)
    acts = _actions(env, 10, n, seed=7)
    perm = rng.permutation(n)
    a = VecEnv(env, n)
    a.set_model_factors(friction=F[:, 0], gear=F[:, 1])
    a.reset(keys)
    b = VecEnv(env, n)
    b.set_model_factors(friction=F[perm, 0], gear=F[perm, 1])
    b.reset(keys[perm])
    _same(_trajectory(a, acts), _trajectory(b, acts[:, torch.as_tensor(perm, device="cuda")]), "permuted", rows_a=perm)


@pytest.mark.parametrize("name", ["hopper", "humanoidrun"])
def test_graph_replay_follows_in_place_rewrites(name):
    """20 replays of a captured step = 20 eager steps; the table is rewritten in place after 10 (same tensor, new values) and both
    follow it, while a third env that keeps the old table does not"""
    env, n = _env(name), 256
    rng = np.random.default_rng(8)
    F0, F1 = (rng.uniform(0.2, 1.8, (n, 2)).astype(np.float32) for _ in range(2))
    keys = prng.split(prng.PRNGKey(9), n)
    acts = _actions(env, 20, n, seed=10)

    def fresh():
        v = VecEnv(env, n)
        v.set_model_factors(friction=F0[:, 0], gear=F0[:, 1])
        v.reset(keys)
        return v

    eager, kept = fresh(), fresh()
    ref, old = [], []
    for t in range(20):
        if t == 10:
            eager.set_model_factors(friction=F1[:, 0], gear=F1[:, 1])
        ref.append(eager.step(acts[t]).raw.detach().cpu().numpy().copy())
        old.append(kept.step(acts[t]).raw.detach().cpu().numpy().copy())
    venv = fresh()
    venv.step(acts[0])   # warm-up outside the capture, then start over
    venv.reset(keys)
    ptr = venv.factors.data_ptr()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            venv.step()
    torch.cuda.current_stream().wait_stream(s)
    for t in range(20):
        if t == 10:
            venv.set_model_factors(friction=F1[:, 0], gear=F1[:, 1])
            assert venv.factors.data_ptr() == ptr
        venv.actions.copy_(acts[t])
        g.replay()
        assert_bit_exact(venv.state.cpu().numpy(), ref[t].reshape(n, -1), f"replay {t}")
    assert not np.array_equal(ref[-1], old[-1]), "the rewrite changed nothing"


# ---- the controllers against a mismatched plant -------------------------------------------------------------------------------
PLANTS = [(1.0, 1.0), (0.5, 1.0), (1.0, 0.7), (1.5, 1.3)]


def mpc_args(env_name, Nsample=256, Hsample=16, Nstep=20, plants=PLANTS):
    return [mbd_mpc.Args(seed=3 * b, env_name=env_name, Nsample=Nsample, Hsample=Hsample, Ndiffuse=10, Nwarm=3, Nstep=Nstep,
                         temp_sample=0.1, plant_friction=f, plant_gear=g, not_render=True, disable_recommended_params=True)
            for b, (f, g) in enumerate(plants)]


def pi_args(env_name, method="mppi", Nstep=20):
    return [pi_mpc.Args(seed=3 * b, env_name=env_name, update_method=method, Nsample=256, Hsample=16, Nrefine=10, Nwarm=3,
                        Nstep=Nstep, sigma_warm=0.7, temp_sample=0.1, plant_friction=f, plant_gear=g, not_render=True,
                        disable_recommended_params=True) for b, (f, g) in enumerate(PLANTS)]


def _assert_result(r, q, what):
    for f in ("actions", "rewards", "states", "rew_hist"):
        assert_bit_exact(getattr(r, f), getattr(q, f), f"{what}: {f}")


@pytest.mark.parametrize("mod,make,env_name", [(mbd_mpc, mpc_args, "hopper"), (mbd_mpc, mpc_args, "humanoidrun"),
                                               (pi_mpc, pi_args, "hopper")], ids=["mbd-hopper", "mbd-humanoidrun", "mppi-hopper"])
def test_graph_replay_equals_the_host_driven_loop(mod, make, env_name):
    """20 control steps of the 4 plants: the device loop (per-env factors in the VecEnv) = the host loop (each problem's plant is its
    scaled_env), bit for bit; the mismatched plants are not the nominal one"""
    al = make(env_name)
    env = mod._prepare(al, batch=True)
    dev = mod.Controller(env, al)
    assert dev.venv.factors is not None
    r = dev.run()
    host = mod.Controller(env, al, host=True)
    assert [bool((p.blob == env.blob).all()) for p in host.plants] == [True, False, False, False]
    _assert_result(r, host.run_host_driven(), env_name)
    assert np.isfinite(r.states).all()
    assert all(not np.array_equal(r.states[b], r.states[0]) for b in range(1, 4))


def test_unit_plant_is_todays_run_mpc():
    al = mpc_args("hopper")
    _, res = mbd_mpc.run_mpc_batch(al, return_result=True)
    _, q = mbd_mpc.run_mpc(mpc_args("hopper")[0], return_result=True)
    for f in ("actions", "rewards", "states", "rew_hist"):
        assert_bit_exact(getattr(res, f)[0], getattr(q, f)[0], f"problem 0: {f}")


@pytest.mark.parametrize("env_name", ["hopper", "humanoidrun"])
def test_control_step_0(env_name):
    """P_0 does not depend on the plant; s_1 and r_0 are the plant's scaled_env.step(s_0, a_0)"""
    al = mpc_args(env_name, Nstep=1)
    env = mbd_mpc._prepare(al, batch=True)
    ctl = mbd_mpc.Controller(env, al)
    res = ctl.run()
    nom = mbd_mpc.Controller(env, mpc_args(env_name, Nstep=1, plants=[(1.0, 1.0)] * 4))
    nres = nom.run()
    assert nom.venv.factors is None
    assert_bit_exact(ctl.engine.Ybars[:, 0].cpu().numpy(), nom.engine.Ybars[:, 0].cpu().numpy(), "P_0")
    assert_bit_exact(res.actions, nres.actions, "a_0")
    for b, (f, g) in enumerate(PLANTS):
        s1 = scaled_env(env, f, g).step(ctl.host_states[b], res.actions[b, 0])
        assert_bit_exact(res.states[b, 0], mbd_mpc.host_raw(env, ctl.host_states[b]), "s_0")
        assert_bit_exact(res.states[b, 1], mbd_mpc.host_raw(env, s1), f"s_1 of plant {b}")
        assert_bit_exact(res.rewards[b, 0], np.float32(s1.reward), f"r_0 of plant {b}")
