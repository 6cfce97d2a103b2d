"""Each CUDA rollout kernel against the float64 reference of one positional substep (tests/xpbd_ref.py), without the
oracle: one launch per constructed state (tests/xpbd_families.py), H = 1, one substep, a ragged batch of actions; then a
second launch at the env's own n_frames whose rewards are checked against the float64 reward of the kernel's own state."""
import numpy as np
import pytest
import torch

from mbd_b200 import ops
from mbd_b200.model import blob as B
from tests import xpbd_families as F
from tests import xpbd_ref as X

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = 2.0
HUMANOIDS = ["humanoidrun", "humanoidstandup", "humanoidtrack"]
OTHERS = ["hopper", "walker2d", "ant", "halfcheetah", "cartpole", "contact_params"] + [f"gen{s}" for s in F.MODELGEN_SEEDS]
CASES = [(m, v) for m in HUMANOIDS for v in (0, 1, 2, 3, 8)] + [(m, v) for m in OTHERS for v in (1, 2)]


def launched_kernel(blob, variant, n, sms):
    """the rollout kernel `choose_kernel` (csrc/mbd_b200.cu) runs for a requested variant: it remaps variants a model cannot
    take (named barriers need 2 per parent within 15, the packed kernel 11 hinge-only links with at most 2 contacts each)"""
    bi = blob.view(np.int32)
    L = int(bi[B.H_NLINK])
    lf = lambda f: bi[B.HDR_WORDS + f * B.MAXL:B.HDR_WORDS + f * B.MAXL + L]   # noqa: E731
    max_ncon = int(lf(B.F_NCON).max())
    named_ok = 2 * int((lf(B.F_CHILD0) >= 0).sum()) <= 15
    pk_ok = L == 11 and not lf(B.F_SLIDE).any() and int(bi[B.H_REWARD]) in (
        B.REWARD_HUMANOIDRUN, B.REWARD_HUMANOIDTRACK, B.REWARD_HUMANOIDSTANDUP, B.REWARD_ANT)
    v = variant
    if v == 0:
        v = (1 if n <= sms * 16 else 3 if n <= sms * 32 else 8 if max_ncon <= 2 and pk_ok else 2) if L == 11 else 2
    if not named_ok and v == 3:
        v = 2
    if v == 8 and not (pk_ok and max_ncon <= 2):
        v = 2
    if v == 8:
        return "pk-group"
    if v == 1:
        return "lane-per-link"
    if L == 11 and v == 2:
        return "wpl-cta"
    if L == 11 and v == 3:
        return "wpl-named"
    return "wpl-generic"


def test_every_rollout_kernel_is_covered(tmp_path):
    """the (model, variant) cases below launch every rollout kernel at least once, after the launcher's remapping"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = {launched_kernel(F.make_env(m, tmp_path).blob, v, 129, sms) for m, v in CASES}
    want = {"lane-per-link", "wpl-cta", "wpl-named", "wpl-generic", "pk-group"}
    assert want <= got, want - got


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=DEV)


def _within(got, ref, what):
    ok = ~ref["undecided"]
    d = np.abs(got.astype(np.float64) - ref["value"])[ok]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / ref["radius"][ok])
    assert q.size == 0 or q.max() <= K, f"{what}: {q.max():.3g} radii"


def _rew_within(got, ref, what):
    d = np.abs(np.asarray(got, np.float64) - ref.v)
    assert np.all(d <= K * ref.r), f"{what}: {np.max(d / ref.r):.3g} radii"


@pytest.mark.parametrize("name,variant", CASES)
def test_kernel_within_the_float64_bound(tmp_path, name, variant):
    env = F.make_env(name, tmp_path)
    m = env.device_model(torch.device(DEV))
    ops.set_kernel_variant(variant)
    try:
        for fam in F.FAMILIES:
            und, tot = 0, 0
            for i, (st, u) in enumerate(F.build(env, fam, 129 if F.FAMILIES.index(fam) % 2 else 77)):
                n = u.shape[0]
                ref = X.positional_step(env.blob, np.broadcast_to(st, (n,) + st.shape), u)
                out = ops.rollout(m, T(st), T(u[:, None]), want_final=True, want_rewss=True, nsub_override=1)
                _within(out["final"].cpu().numpy(), ref, f"{name} v{variant} {fam}[{i}]")
                und, tot = und + int(ref["undecided"].sum()), tot + n
            assert und <= F.undecided_cap(name, fam) * max(tot, 1), f"{name} {fam}: {und} of {tot} samples undecided"
            if fam != "F1":
                continue
            # rewards at the env's own n_frames, against the float64 reward of the kernel's own final state
            st, u = F.build(env, "F1", 77)[0]
            kind = int(env.blob.view(np.int32)[B.H_REWARD])
            xref = T(env.xref) if name == "humanoidtrack" else None
            out = ops.rollout(m, T(st), T(u[:, None]), xref=xref, want_final=True, want_rewss=True, want_track=xref is not None)
            fin = out["final"].cpu().numpy()
            rew = out["rewss"].cpu().numpy()[:, 0]
            sts = np.broadcast_to(st, (u.shape[0],) + st.shape)
            if kind == B.REWARD_HUMANOIDTRACK:
                _rew_within(rew, X.reward_pre(env.blob, sts), "reward_pre")
                tv, tr = X.track_positions(env.blob, fin)
                tk = out["track"].cpu().numpy()[:, 0]
                assert np.all(np.abs(tk - tv) <= K * tr), "tracked positions"
                _rew_within(out["logpd"].cpu().numpy(), X.logpd_one_step(env.blob, fin, env.xref[:, 0]), "logpd")
            elif kind == B.REWARD_ANT:
                _rew_within(rew, X.reward_ant(env.blob, sts, fin, u), "ant reward")
            else:
                _rew_within(rew, X.reward_post(env.blob, fin), "reward_post")
    finally:
        ops.set_kernel_variant(0)
