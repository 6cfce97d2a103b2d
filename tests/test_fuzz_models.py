"""Differential tests on RANDOM models (tests/modelgen.py): the model compiler, the CPU oracle and every rollout-kernel mapping
must agree on kinematic trees nobody hand-tuned — 1..16 links, up to 4 children, one or two world-parented trees, free / planar /
sliding / hinge-only roots, 1..3 stacked hinges about arbitrary orthonormal axes, joints that start outside their range,
0..6 plane contacts per link.  The fixed envs only cover the shapes the reference happens to ship
(upstream mbd/envs/__init__.py:9-33); the generic path (`GenericPositionalEnv`, `k_rollout_wpl<..., L != 11>`) is what a
user's own MJCF runs on."""
import numpy as np
import pytest

import mbd_b200
from mbd_b200 import prng

from tests.conftest import assert_bit_exact
from tests import modelgen

SEEDS = list(range(48))
SEEDS11 = list(range(100, 124))   # random 11-link trees: the link count the specialised kernels (named barriers, two-group, packed) are built for


def _env(tmp_path, seed, n_frames=3, links=0, topology=""):
    xml, facts = modelgen.random_model(seed, links=links, topology=topology)
    p = tmp_path / f"fuzz_{seed}.xml"
    p.write_text(xml)
    return mbd_b200.envs.GenericPositionalEnv(str(p), n_frames=n_frames), facts


def _actions(seed, n, H, nu):
    rng = np.random.default_rng(1000 + seed)
    return np.clip(rng.normal(size=(n, H, nu)).astype(np.float32) * 0.7, -1.0, 1.0)


def test_generator_is_deterministic_and_covers_the_subset():
    facts = [modelgen.random_model(s)[1] for s in SEEDS]
    assert modelgen.random_model(5)[0] == modelgen.random_model(5)[0]
    assert any(f["roots"] == 2 for f in facts) and any(f["max_children"] == 4 for f in facts)
    assert min(f["L"] for f in facts) == 1 and max(f["L"] for f in facts) == 16
    assert any(f["ncon"] == 0 for f in facts) and max(f["ncon"] for f in facts) > 16
    xmls = "".join(modelgen.random_model(s)[0] for s in SEEDS)
    for needle in ('type="free"', 'type="slide"', 'limited="false"', 'range="10 ', 'type="capsule"', 'type="sphere"', " ref="):
        assert needle in xmls, needle


@pytest.mark.parametrize("seed", SEEDS)
def test_compile_and_oracle_on_random_models(orc, tmp_path, seed):
    """host logic: MJCF -> system -> blob; reset (FK) and obs (IK) are inverse; the oracle rollout is reproducible and its
    one-sample result does not depend on which other samples share the call"""
    env, facts = _env(tmp_path, seed)
    sys_ = env.sys
    assert sys_.num_links() == facts["L"] and env.action_size == facts["nu"]
    st = env.reset(prng.split(prng.PRNGKey(seed))[1])
    raw = st.pipeline_state.raw
    assert raw.shape == (facts["L"], 13) and np.isfinite(raw).all()
    # FK / IK round trip on perturbed joint coordinates (small angles: no wrap-around)
    rng = np.random.default_rng(seed)
    q = sys_.init_q.copy()
    hinge_or_slide = np.ones(q.size, dtype=bool)       # free-joint coordinates (pos + unit quaternion) are left alone
    for l in range(facts["L"]):
        if sys_.link_types[l] == "f":
            hinge_or_slide[int(sys_.link_q_start[l]):int(sys_.link_q_start[l]) + 7] = False
    q[hinge_or_slide] += rng.uniform(-0.1, 0.1, size=int(hinge_or_slide.sum()))
    qd = rng.uniform(-0.5, 0.5, size=sys_.qd_size())
    ps = env.pipeline_init(q, qd)
    np.testing.assert_allclose(ps.q[hinge_or_slide], q[hinge_or_slide], atol=5e-5)
    # rates: the inverse projects the relative angular velocity on the instantaneous axes (mbd_b200/model/kinematics.py::inverse),
    # which inverts the forward map only where the axes are orthogonal — check the single-dof links
    one = [int(sys_.link_dof_start[l]) for l in range(facts["L"]) if sys_.link_types[l] == "1"]
    np.testing.assert_allclose(ps.qd[one], qd[one], atol=5e-4)
    if facts["nu"] == 0:
        return
    Y = _actions(seed, 5, 4, facts["nu"])
    a = orc.xpbd_rollout(env.blob, raw, Y, want_rewss=True, want_final=True)
    b = orc.xpbd_rollout(env.blob, raw, Y[3:4], want_rewss=True, want_final=True)
    assert_bit_exact(a["final"][3:4], b["final"], "sample independence")
    assert_bit_exact(a["rewss"][3:4], b["rewss"], "sample independence (rewards)")


def _check_all_variants(orc, env, facts, seed, n=77, H=6):
    import torch
    from mbd_b200 import ops
    dev = torch.device("cuda:0")
    raw = env.reset(prng.split(prng.PRNGKey(seed))[1]).pipeline_state.raw
    Y = _actions(seed, n, H, facts["nu"])
    ref = orc.xpbd_rollout(env.blob, raw, Y, want_rewss=True, want_final=True)
    if not (np.isfinite(ref["final"]).all() and np.isfinite(ref["rewss"]).all()):
        pytest.skip("the random model diverges to non-finite values (NaN payloads are not comparable)")
    m = env.device_model(dev)
    st_d = torch.as_tensor(raw, device=dev)
    Y_d = torch.as_tensor(Y, device=dev)
    for v in (0, 1, 2, 3, 8):
        ops.set_kernel_variant(v)
        try:
            out = ops.rollout(m, st_d, Y_d, want_rewss=True, want_final=True)
        finally:
            ops.set_kernel_variant(0)
        assert_bit_exact(out["final"].cpu().numpy(), ref["final"], f"seed {seed} variant {v} final")
        assert_bit_exact(out["rewss"].cpu().numpy(), ref["rewss"], f"seed {seed} variant {v} rewss")
        assert_bit_exact(out["rews"].cpu().numpy(), ref["rews"], f"seed {seed} variant {v} rews")


@pytest.mark.gpu
@pytest.mark.parametrize("topology,seed", [("chain", 200), ("chain", 201), ("chain", 202), ("lonely", 210), ("lonely", 211), ("lonely", 212)])
def test_rollout_kernels_on_the_topologies_the_barrier_protocols_special_case(orc, tmp_path, topology, seed):
    """11-link models the specialised kernels must either handle or hand back to the generic one:
    * "chain": ten links with children need 20 named barriers, the hardware has 15 -> the library falls back to CTA barriers
      (launching the named-barrier kernel anyway would use invalid barrier ids);
    * "lonely": a single-link free body with contacts is a 'late leaf' of the group-barrier protocol although it has no joint —
      host-side count and device-side predicate must agree or the group barrier never completes."""
    env, facts = _env(tmp_path, seed, links=11, topology=topology)
    _check_all_variants(orc, env, facts, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS + SEEDS11)
def test_rollout_kernels_match_oracle_on_random_models(orc, tmp_path, seed):
    """every kernel mapping (auto, lane-per-link, warp-per-link with CTA / named barriers, packed two-sample with group barriers;
    variants that do not apply to a model fall back inside the library) == oracle, bit for bit, on a ragged sample count
    (77: two full 32-sample groups and a partial one; one full and one partial 64-sample packed CTA)"""
    env, facts = _env(tmp_path, seed, links=11 if seed >= 100 else 0)
    if facts["nu"] == 0:
        pytest.skip("model without actuators")
    _check_all_variants(orc, env, facts, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 3, 17, 26])
def test_diffusion_step_on_random_models(orc, tmp_path, seed):
    """the whole reverse step (sampling + rollouts + statistics + weighted mean + update) on a random model vs the oracle
    planner: per-sample quantities bit-exact, reduced outputs to rtol 1e-4 (summation order differs, DESIGN.md §3)"""
    import torch
    from mbd_b200.planners import engine as eng
    from oracle import planner as oplanner
    env, facts = _env(tmp_path, seed)
    dev = torch.device("cuda:0")
    raw = env.reset(prng.split(prng.PRNGKey(seed))[1]).pipeline_state.raw
    H, n = 5, 128
    _, alphas, alphas_bar, sigmas = eng.make_schedule(1e-4, 1e-2, 20)
    e = eng.DiffusionEngine(env, n, H, 0.1, False, raw)
    key = np.uint32([7, seed])
    Ybar = (np.random.default_rng(seed).normal(size=(H, facts["nu"])) * 0.1).astype(np.float32)
    o, rew = e.reverse_once(key, float(sigmas[12]), torch.as_tensor(Ybar.reshape(-1), device=dev), eng.update_coef(alphas, alphas_bar, 12))
    oenv = oplanner.OracleEnv("xpbd", facts["nu"], blob=env.blob, state=raw)
    ref = oplanner.reverse_once(oenv, key, n, H, float(sigmas[12]), Ybar.reshape(-1), 0.1, alphas, alphas_bar, 12)
    if not np.isfinite(ref["rews"]).all():
        pytest.skip("the random model diverges to non-finite values")
    assert_bit_exact(e.rews_local.cpu().numpy(), ref["rews"], f"seed {seed} per-sample returns")
    assert_bit_exact(e.Y0s.cpu().numpy(), ref["Y0s"], f"seed {seed} sampled actions")
    scale = max(np.abs(ref["Ybar_im1"]).max(), 1e-6)
    assert np.abs(o.cpu().numpy() - ref["Ybar_im1"]).max() / scale < 1e-4
    assert abs(rew.item() - ref["rew_mean"]) <= 1e-4 * max(abs(ref["rew_mean"]), 1e-6) + 1e-6
    # the same step sharded over two emulated ranks (64 samples each: whole runs -> the single-rank bits)
    keys = np.zeros((20, 2), np.uint32); keys[12] = key
    ranks = eng.DiffusionEngine.make_emulated_ranks(env, n, H, 0.1, False, raw, 2, Ndiffuse=20)
    for r in ranks:
        r.load_schedule(keys, sigmas, alphas, alphas_bar); r.set_step(12)
        r.Ybars[12].copy_(torch.as_tensor(Ybar.reshape(-1), device=dev))
    eng.DiffusionEngine.step_emulated_ranks(ranks)
    torch.cuda.synchronize()
    for r in ranks:
        r.check_exchange()
        assert_bit_exact(r.Ybars[11].cpu().numpy(), o.cpu().numpy(), f"seed {seed}: rank {r.rank} of 2 vs one rank")
    assert_bit_exact(np.concatenate([r.rews_local.cpu().numpy() for r in ranks]), ref["rews"], f"seed {seed}: sharded returns")
