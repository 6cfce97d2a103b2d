"""The RL kernels on the device against the float64 reference with a radius per value (tests/rl_ref.py), on the families of
tests/rl_families.py, at the launch shapes where their loops change (DESIGN.md §2, "Accuracy contract of the RL acting step, GAE
and statistics"): k_ppo_act at B = 1, 33 and 8 * 4 * SMs + 37 (two grid-stride passes), k_sac_act at B = 1 and 7 (mod 8),
k_ppo_gae at mb from 1 to 4096 and T in {1, 5, 20} (one shape whose noise loop iterates), k_ppo_stat_* at 1, 256, 257 and 301
chunks with O in {1, 128} and over a count past 2^24, and k_sac_record with its grid-stride loop.  Where bit equality with the
host harness, `ppo_ref.gae_kernel_f32`, `normal_host` or `sac_ref.RingRef` is defined, it is asserted too."""
import numpy as np
import pytest
import torch

from mbd_b200 import _lib, ops, prng
from mbd_b200.blackbox.mbd_mnist import normal_host
from tests import ppo_ref, sac_ref
from tests import rl_families as F
from tests import rl_ref as X
from tests.test_ppo_cpu import harness, host_act  # noqa: F401  (harness: the fixture of the host build)
from tests.test_rl_ref_cpu import GAE_SHAPES, K, ROWS, check_act, gae_check
from tests.test_sac_cpu import host_act as sac_host_act
from tests.test_sac_cpu import sac_harness  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _t(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV) if dtype is None else torch.zeros(a, dtype=dtype, device=DEV)


def _bits(a, b, what):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), \
        f"{what}: {np.count_nonzero(a.view(np.uint32) != b.view(np.uint32))} of {a.size} differ"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ppo_act_dev(O, nu, pol, mean, std, obs, key):
    """one MBD_PPO_ACT launch on a plan of its own: (actions, raw, logp)"""
    B = obs.shape[0]
    f = torch.float32
    keep = dict(pol=_t(pol), mean=_t(mean), std=_t(std), obs=_t(obs), keys=_t(key.reshape(1, 2).view(np.int32)),
                ctl=_t((4,), torch.int32), er=_t((B,), f), ed=_t((B,), f), et=_t((B,), f), act=_t((B, nu), f),
                rec=_t((2, B, O), f), raw=_t((1, B, nu), f), logp=_t((1, B), f), rw=_t((1, B), f), dc=_t((1, B), f), tr=_t((1, B), f))
    P = _lib.PpoPlan()
    P.B, P.O, P.nu, P.slots, P.unroll, P.mb, P.act_key_rows, P.loss_key_rows = B, O, nu, 1, 1, 1, 1, 1
    for field, k in (("policy_dev", "pol"), ("mean_dev", "mean"), ("std_dev", "std"), ("act_keys_dev", "keys"), ("act_ctl_dev", "ctl"),
                     ("env_obs_dev", "obs"), ("env_reward_dev", "er"), ("env_done_dev", "ed"), ("env_trunc_dev", "et"),
                     ("env_actions_dev", "act"), ("obs_dev", "rec"), ("raw_dev", "raw"), ("logp_dev", "logp"), ("reward_dev", "rw"),
                     ("disc_dev", "dc"), ("trunc_dev", "tr")):
        setattr(P, field, keep[k].data_ptr())
    ops.ppo_act(P, _lib.PPO_ACT)
    torch.cuda.synchronize()
    assert keep["ctl"].cpu().tolist() == [1, 1, 0, 0]
    return keep["act"].cpu().numpy(), keep["raw"][0].cpu().numpy(), keep["logp"][0].cpu().numpy()


def sac_act_dev(O, nu, pol, mean, std, obs, key):
    """one MBD_SAC_ACT launch: (actions, ring rows)"""
    B = obs.shape[0]
    f = torch.float32
    R = 2 * O + nu + 3
    keep = dict(pol=_t(pol), mean=_t(mean), std=_t(std), obs=_t(obs), keys=_t(key.reshape(1, 2).view(np.int32)),
                ctl=_t((4,), torch.int32), rctl=_t((4,), torch.int32), act=_t((B, nu), f), stage=_t((B, O), f), ring=_t((B, R), f))
    P = _lib.SacPlan()
    P.B, P.O, P.nu, P.capacity, P.batch, P.updates, P.act_key_rows, P.noise_key_rows = B, O, nu, B, 1, 1, 1, 1
    for field, k in (("policy_dev", "pol"), ("mean_dev", "mean"), ("std_dev", "std"), ("act_keys_dev", "keys"), ("act_ctl_dev", "ctl"),
                     ("env_obs_dev", "obs"), ("env_actions_dev", "act"), ("stage_obs_dev", "stage"), ("ring_dev", "ring"),
                     ("ring_ctl_dev", "rctl")):
        setattr(P, field, keep[k].data_ptr())
    ops.sac_act(P, _lib.SAC_ACT)
    torch.cuda.synchronize()
    return keep["act"].cpu().numpy(), keep["ring"].cpu().numpy()


def _report(tag, worst):
    print(f"{tag:32s} largest |kernel - f64| / radius {({k: round(v, 3) for k, v in worst.items()})}")


@pytest.mark.parametrize("Bsel", ["1", "33", "two_passes"])
def test_ppo_act_within_the_bound(harness, Bsel):  # noqa: F811
    B = {"1": 1, "33": 33, "two_passes": 8 * 4 * _sms() + 37}[Bsel]
    if Bsel == "two_passes":
        grid = min(-(-B // 8), 4 * _sms())          # mbd_ppo_act's launch: 8 warps (envs) per CTA, at most 4 CTAs per SM
        assert grid * 8 < B, "the grid-stride loop of k_ppo_act runs once only"
    shapes = [(128, 32), (33, 17)] if B > 1000 else None
    for fam, cases in F.act_cases("ppo", B, shapes=shapes).items():
        worst = {}
        for case in cases:
            got = ppo_act_dev(*case)
            O, nu, pol, mean, std, obs, key = case
            want = host_act(harness, pol, mean, std, obs, normal_host(key, (B, nu)))
            for g, w, n in zip(got, want, ("actions", "raw", "logp")):
                _bits(g, w, f"{fam} O={O} nu={nu} {n} vs the host harness")
            r, _ = check_act("ppo", case, got, f"k_ppo_act B={B} {fam}")
            worst = {k: max(worst.get(k, 0.0), v) for k, v in r.items()}
        _report(f"k_ppo_act B={B} {fam}", worst)


@pytest.mark.parametrize("B", [1, 1031])
def test_sac_act_within_the_bound(sac_harness, B):  # noqa: F811
    shapes = [(128, 32), (11, 3)] if B > 1000 else None
    for fam, cases in F.act_cases("sac", B, shapes=shapes).items():
        worst = {}
        for case in cases:
            act, ring = sac_act_dev(*case)
            O, nu, pol, mean, std, obs, key = case
            a_h, raw_h, lp_h = sac_host_act(sac_harness, pol, mean, std, obs, normal_host(key, (B, nu)))
            _bits(act, a_h, f"{fam} O={O} nu={nu} actions vs the host harness")
            _bits(ring[:, O:O + nu], a_h, "ring actions")
            _bits(ring[:, :O], obs, "ring obs")
            r, _ = check_act("sac", case, (act, raw_h, lp_h), f"k_sac_act B={B} {fam}")
            worst = {k: max(worst.get(k, 0.0), v) for k, v in r.items()}
        _report(f"k_sac_act B={B} {fam}", worst)


# ---- GAE --------------------------------------------------------------------------------------------------------------------------
def gae_dev(c, nu=2, key_seed=5):
    T, mb, B = c["T"], c["mb"], c["B"]
    f = torch.float32
    keep = dict(rw=_t(c["reward"]), dc=_t(c["disc"]), tr=_t(c["trunc"]), traj=_t(c["traj"]), vals=_t(c["values"]),
                vs=_t((T, mb), f), adv=_t((T, mb), f), ent=_t((T, mb, nu), f),
                keys=_t(prng.PRNGKey(key_seed).reshape(1, 2).view(np.int32)), lctl=_t((1,), torch.int32))
    P = _lib.PpoPlan()
    P.B, P.O, P.nu, P.slots, P.unroll, P.mb, P.act_key_rows, P.loss_key_rows = B, 1, nu, T, T, mb, 1, 1
    P.reward_scaling, P.discount, P.gae_lambda = c["reward_scaling"], c["discount"], c["lam"]
    for field, k in (("reward_dev", "rw"), ("disc_dev", "dc"), ("trunc_dev", "tr"), ("traj_dev", "traj"), ("values_dev", "vals"),
                     ("vs_dev", "vs"), ("adv_dev", "adv"), ("ent_eps_dev", "ent"), ("loss_keys_dev", "keys"), ("loss_ctl_dev", "lctl")):
        setattr(P, field, keep[k].data_ptr())
    ops.ppo_gae(P)
    torch.cuda.synchronize()
    return keep["vs"].cpu().numpy(), keep["adv"].cpu().numpy(), keep["ent"].cpu().numpy()


def test_gae_within_the_bound():
    worst = {}
    for fam in F.GAE_FAMILIES:
        for k, (T, mb) in enumerate(GAE_SHAPES):
            for Tt in sorted({T, 1, 20}) if fam == "mild" else (T,):
                c = F.gae_case(fam, Tt, mb, seed=k, params=F.GAE_PARAMS[k % len(F.GAE_PARAMS)])
                vs, adv, _ = gae_dev(c)
                vs32, adv32 = ppo_ref.gae_kernel_f32(c["reward"], c["disc"], c["trunc"], c["values"], c["traj"], c["B"], c["T"],
                                                     c["reward_scaling"], c["discount"], c["lam"])
                _bits(vs, vs32, f"{fam} T={Tt} mb={mb} vs")
                _bits(adv, adv32, f"{fam} T={Tt} mb={mb} advantages")
                qv, qa, *_ = gae_check(c, vs, adv)
                assert qv <= K and qa <= K, f"{fam} T={Tt} mb={mb}: vs {qv:.3g}, advantages {qa:.3g} radii"
                w = worst.setdefault(fam, [0.0, 0.0])
                w[0], w[1] = max(w[0], qv), max(w[1], qa)
    for fam, (a, b) in worst.items():
        print(f"k_ppo_gae {fam:12s} largest ratio vs {a:.3f}  normalised advantages {b:.3f}")


def test_gae_noise_loop_iterates():
    """T * mb * Nu above 264 CTAs x 1024 threads: the noise loop takes a second pass; bit for bit against normal_host"""
    T, mb, nu = 20, 4096, 4
    assert T * mb * nu > 264 * 1024
    c = F.gae_case("mild", T, mb)
    _, _, ent = gae_dev(c, nu=nu, key_seed=9)
    _bits(ent, normal_host(prng.PRNGKey(9), (T, mb, nu)), "entropy noise")


# ---- statistics -------------------------------------------------------------------------------------------------------------------
def stats_dev(O, B, slots, batches):
    """mbd_ppo_obs_stats over each batch [slots * B][O] in turn: [(stat state, mean, std)] after every update"""
    rows = slots * B
    chunks = -(-rows // ROWS)
    f = torch.float32
    keep = dict(obs=_t((slots, B, O), f), stat=_t((1 + 2 * O,), torch.float64), scr=_t((chunks * 2 * O,), torch.float64),
                mean=_t((O,), f), std=_t((O,), f))
    P = _lib.PpoPlan()
    P.B, P.O, P.nu, P.slots, P.unroll, P.mb = B, O, 1, slots, 1, 1
    for field, k in (("obs_dev", "obs"), ("stat_dev", "stat"), ("stat_scratch_dev", "scr"), ("mean_dev", "mean"), ("std_dev", "std")):
        setattr(P, field, keep[k].data_ptr())
    out = []
    for x in batches:
        keep["obs"].copy_(torch.from_numpy(x.reshape(slots, B, O)))
        ops.ppo_obs_stats(P)
        torch.cuda.synchronize()
        out.append((keep["stat"].cpu().numpy().copy(), keep["mean"].cpu().numpy().copy(), keep["std"].cpu().numpy().copy()))
    return out, chunks


STAT_LAUNCHES = [(1, 200, 1), (128, 65536, 1), (1, 21871, 3), (128, 21871, 3), (1, 38437, 2), (128, 38437, 2)]   # (O, B, slots)


def test_stats_within_the_bound():
    worst = {}
    for fam in F.STAT_FAMILIES:
        launches = [(1, 65536, 16)] if fam == "count" else STAT_LAUNCHES
        for O, B, slots in launches:
            batches = F.stat_batches(fam, O, B * slots, 17 if fam == "count" else 3)
            got, chunks = stats_dev(O, B, slots, batches)
            st = (0.0, np.zeros(O), np.zeros(O))
            for x, (stat, mean32, std32) in zip(batches, got):
                st, ref = X.stats_update(st, x, chunks)
                assert stat[0] == st[0]
                q = max(float(X.ratio(mean32, ref["mean"]).max()), float(X.ratio(std32, ref["std"]).max()))
                assert q <= K, f"{fam} O={O} chunks={chunks}: {q:.3g} radii (mean {mean32[:3]} vs {ref['mean'].v[:3]}, std " \
                               f"{std32[:3]} vs {ref['std'].v[:3]})"
                assert np.all(np.abs(stat[1:1 + O] - st[1]) <= 2 * ref["state_mean_r"] + 1e-300)
                assert np.all(np.abs(stat[1 + O:] - st[2]) <= 2 * ref["state_sv_r"] + 1e-300)
                worst[(fam, chunks)] = max(worst.get((fam, chunks), 0.0), q)
            if fam == "count":
                assert st[0] > 2 ** 24
    for (fam, chunks), q in sorted(worst.items()):
        print(f"k_ppo_stat {fam:9s} chunks {chunks:4d} largest ratio {q:.3f}")


# ---- the replay record ------------------------------------------------------------------------------------------------------------
def test_sac_record_grid_stride_matches_the_ring():
    O, nu, B, cap = 128, 6, 2100, 5000
    assert B * (O + 3) > 1024 * 256          # mbd_sac_record launches at most 1024 CTAs of 256 threads
    R = 2 * O + nu + 3
    rng = np.random.default_rng(0)
    data = rng.normal(size=(cap, R)).astype(np.float32)
    pos, size = 4000, 4500
    obs = rng.normal(size=(B, O)).astype(np.float32)
    rew, done = rng.normal(size=B).astype(np.float32), (rng.uniform(size=B) < 0.2).astype(np.float32)
    trunc = done * (rng.uniform(size=B) < 0.5).astype(np.float32)
    keep = dict(ring=_t(data), rctl=_t(np.array([pos, size, 0, 0], np.int32)), obs=_t(obs), rw=_t(rew), dn=_t(done), tr=_t(trunc))
    P = _lib.SacPlan()
    P.B, P.O, P.nu, P.capacity, P.batch, P.updates = B, O, nu, cap, 1, 1
    for field, k in (("ring_dev", "ring"), ("ring_ctl_dev", "rctl"), ("env_obs_dev", "obs"), ("env_reward_dev", "rw"),
                     ("env_done_dev", "dn"), ("env_trunc_dev", "tr")):
        setattr(P, field, keep[k].data_ptr())
    ops.sac_record(P)
    torch.cuda.synchronize()
    ring = sac_ref.RingRef(cap, R)
    ring.data[:], ring.pos, ring.size = data, pos, size
    rows = data[(pos + np.arange(B)) % cap].copy()
    rows[:, O + nu], rows[:, O + nu + 1], rows[:, O + nu + 2:2 * O + nu + 2], rows[:, 2 * O + nu + 2] = rew, 1 - done, obs, trunc
    ring.insert(rows)
    _bits(keep["ring"].cpu().numpy(), ring.data, "ring")
    assert keep["rctl"].cpu().tolist() == [ring.pos, ring.size, 0, 0]
