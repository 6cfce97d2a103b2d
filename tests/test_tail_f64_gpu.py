"""The tail of a diffusion step (k_step_weights + k_step_update, driven through mbd_step_tail_launch with constructed
returns and samples) and the round-1 kernels the path-integral planners use (k_softmax_weights, k_wsum_runs, k_wsum_tree,
k_update), against the float64 reference of tests/tail_ref.py — per weight, per column, at the tiling edges of the kernels:
the 8192-thread cluster stride, 64-sample runs, the 32-row / 8-row / single-row paths of the pairwise tree over the runs,
256-column blocks up to the 27-block cap, and rank boundaries (P emulated ranks on one device, one stream each).

Exact checks where the arithmetic is exact: one overwhelming sample gets weight 1.0f and the iterate is the fp32 update of
its row bit for bit, wherever that sample sits; an exact two-way tie gets 0.5f / 0.5f.

GPU memory: the largest cases hold 2553 x 6912, 65536 x 257 and 8 x 4159 x 1020 samples, i.e. 71 MB, 67 MB and 136 MB of
Y0s plus the run scratch (under 10 % of that); the extremes (65536 samples, 6912 columns) are not combined."""
import math

import numpy as np
import pytest
import torch

import mbd_b200
from mbd_b200 import _lib, ops
from mbd_b200.planners import engine as eng
from tests import tail_ref as tr
from tests.conftest import assert_bit_exact

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
f32 = np.float32
TEMPS = (0.01, 0.1, 1.0, 5.0)
BIG = f32(50.0)          # a sentinel return: every other log-weight lands below -87 at temp 0.01


def _rig(N, HNu, P, demo=False):
    """engines without an env, Nu = 1 so that H * Nu can be any column count; a demo tail needs a demonstration, of which it
    reads nothing"""
    inputs = eng.LaunchInputs(xref=torch.zeros((4, 2), device=DEV)) if demo else eng.LaunchInputs.none()
    if P == 1:
        return [eng.DiffusionEngine(None, N, HNu, 0.1, demo, None, device=DEV, inputs=inputs, nu=1)]
    return eng.DiffusionEngine.make_emulated_ranks(None, N, HNu, 0.1, demo, None, P, device=DEV, inputs=inputs, nu=1)


def _load(engines, rews=None, Y=None, Ybar_i=None, coef=None, logpd=None):
    for e in engines:
        sl = slice(e.n_begin, e.n_begin + e.n_local)
        if Y is not None:
            e.Y0s.copy_(torch.from_numpy(np.ascontiguousarray(Y[sl])))
        if rews is not None:
            e.rews_local.copy_(torch.from_numpy(np.ascontiguousarray(rews[sl])))
        if logpd is not None:
            e.logpd_local.copy_(torch.from_numpy(np.ascontiguousarray(logpd[sl])))
        if coef is not None:
            e.stage_step(np.zeros(2, np.uint32), 0.0, torch.from_numpy(Ybar_i).to(DEV), coef, 1)


def _tail(engines, temp=None, rew_xref=None):
    """launches 2 and 3 of step 1 on every rank (own stream per rank) and returns the host copies of the outputs"""
    for e in engines:
        e.set_step(1)
        if temp is not None:
            e._plan_c.temp = float(temp)
        if rew_xref is not None:
            e._plan_c.rew_xref = float(rew_xref)
    cur = torch.cuda.current_stream()
    if len(engines) == 1:
        ops.step_tail_launch(engines[0]._plan_c)
    else:
        for e in engines:
            e.stream.wait_stream(cur)
        for e in engines:
            with torch.cuda.stream(e.stream):
                ops.step_tail_launch(e._plan_c)
        for e in engines:
            cur.wait_stream(e.stream)
    torch.cuda.synchronize()
    for e in engines:
        e.check_exchange()
        assert int(e.ctl[0].item()) == 0
    out = dict(w=np.concatenate([e.weights.cpu().numpy() for e in engines]),
               Ybar_im1=[e.Ybars[0].cpu().numpy() for e in engines],
               scalars=engines[0].scalars.cpu().numpy(), rew_hist=engines[0].rew_hist[1].item())
    for e in engines[1:]:
        assert_bit_exact(e.Ybars[0].cpu().numpy(), out["Ybar_im1"][0], f"rank {e.rank} disagrees on the iterate")
        assert_bit_exact(e.scalars.cpu().numpy(), out["scalars"], f"rank {e.rank} disagrees on the statistics")
    return out


def _check(out, f, Y, Ybar_i, coef, temp, N, P, what):
    ref = tr.reference(f["rews"], temp, f["logpd"], f["rew_xref"], Y, Ybar_i, coef)
    sc = out["scalars"]
    assert out["rew_hist"] == float(sc[0]), f"{what}: rew_hist[i] is not the mean of the step"
    wb = tr.check_step(ref, rews=f["rews"], Y0s=Y, Ybar_i=Ybar_i, coef=coef, mean_used=sc[0], std_used=sc[1],
                       weights=out["w"], Ybar_im1=out["Ybar_im1"][0], depth=tr.cluster_depth(N),
                       nruns=math.ceil(N / P / 64), P=P, logpd=f["logpd"], rew_xref=f["rew_xref"], what=what)
    # scalars[3] = sum of exp(logp - max): relative to the float64 sum within the bound of S
    assert abs(float(sc[3]) - ref["S"]) <= wb["sigma_S"] * ref["S"] + 1e-30, f"{what}: sum of exponentials {sc[3]} vs {ref['S']}"
    return ref


# ---- shapes: every tiling edge, normal returns ---------------------------------------------------------------------------

SHAPES = [  # (P, N, HNu): nruns = ceil(N / P / 64) covers 1, 7, 8, 9, 31, 32, 33, 40, 65 and the 32-row blocks beyond
    (1, 1, 1), (1, 2, 255), (1, 63, 256), (1, 64, 257), (1, 65, 850), (1, 443, 1020), (1, 512, 6912), (1, 575, 257),
    (1, 1023, 256), (1, 1025, 255), (1, 1983, 850), (1, 2048, 1), (1, 2112, 1020), (1, 2553, 6912), (1, 4159, 257),
    (1, 7169, 850), (1, 8191, 256), (1, 8192, 1020), (1, 8193, 255), (1, 16389, 1020), (1, 65536, 257),
    (2, 128, 256), (2, 4096, 850), (3, 21, 1), (3, 1725, 257), (5, 325, 6912), (5, 12765, 255), (8, 33272, 1020),
    (8, 65536, 256),
]


@pytest.mark.parametrize("P,N,HNu", SHAPES, ids=[f"P{p}-N{n}-HNu{h}" for p, n, h in SHAPES])
def test_tail_shapes_within_f64_bounds(P, N, HNu):
    temp = TEMPS[(N + HNu) % 4]
    f = tr.make_family("normal", N)
    Y, Ybar_i = tr.make_samples(N, HNu)
    coef = tr.schedule_coef(1 + N % 98)
    engines = _rig(N, HNu, P)
    _load(engines, f["rews"], Y, Ybar_i, coef)
    out = _tail(engines, temp)
    _check(out, f, Y, Ybar_i, coef, temp, N, P, f"P={P} N={N} HNu={HNu} temp={temp}")
    nl = N // P
    if P > 1 and nl % 64 == 0 and ((nl // 64) & (nl // 64 - 1)) == 0:
        # every rank holds 64 * 2^k samples: the sharded tree is a subtree of the single-rank one -> identical bits
        one = _rig(N, HNu, 1)
        _load(one, f["rews"], Y, Ybar_i, coef)
        o1 = _tail(one, temp)
        assert_bit_exact(out["Ybar_im1"][0], o1["Ybar_im1"][0], f"{P} ranks vs one rank: iterate")
        assert_bit_exact(out["w"], o1["w"], f"{P} ranks vs one rank: weights")


# ---- input families ------------------------------------------------------------------------------------------------------

FAMILY_RIGS = [(1, 8193, 257), (3, 8199, 255), (8, 8200, 64)]


@pytest.mark.parametrize("P,N,HNu", FAMILY_RIGS, ids=[f"P{p}-N{n}" for p, n, _ in FAMILY_RIGS])
@pytest.mark.parametrize("fam", tr.FAMILIES)
def test_tail_families_within_f64_bounds(fam, P, N, HNu):
    demo = fam.startswith("demo")
    # the tie sits in cluster CTA 0 and in the last CTA / on the last rank
    f = tr.make_family(fam, N, tie=(5, N - 1))
    Y, Ybar_i = tr.make_samples(N, HNu, seed=1)
    coef = tr.schedule_coef(30)
    engines = _rig(N, HNu, P, demo)
    _load(engines, f["rews"], Y, Ybar_i, coef, f["logpd"])
    for temp in TEMPS:
        out = _tail(engines, temp, f["rew_xref"])
        _check(out, f, Y, Ybar_i, coef, temp, N, P, f"{fam} P={P} N={N} temp={temp}")
        if fam == "constant":
            assert float(out["scalars"][1]) == 1.0 and np.ptp(out["w"]) == 0.0, "constant returns: guarded std, uniform weights"
        if fam == "tie":
            assert out["w"][5] == out["w"][N - 1] and int(np.argmax(out["w"])) == 5, "tied samples must get the same weight"


# ---- sentinels and exact ties: bit-exact wherever the sample sits ---------------------------------------------------------

def _sentinel_positions(N, P):
    nl = N // P
    pos = {0, N - 1, 63, 64, 65, 1023, 1024, 7168, 7175, 7680, 8191, 8192, 15360, 16383, 16384, N - 65}
    for r in range(P):
        pos |= {r * nl, r * nl + nl - 1}
        if nl % 64:
            pos.add(r * nl + (nl // 64) * 64)          # first sample of the ragged last run of rank r
    return sorted(p for p in pos if 0 <= p < N)


SENTINEL_RIGS = [(1, 8193), (1, 16389), (3, 8193), (5, 20795), (8, 8200), (1, 65536)]


@pytest.mark.parametrize("P,N", SENTINEL_RIGS, ids=[f"P{p}-N{n}" for p, n in SENTINEL_RIGS])
def test_tail_sentinel_and_ties_are_exact(P, N):
    HNu = 257                                             # two column blocks, the second one holding a single column
    base = tr.make_family("normal", N)["rews"]
    Y, Ybar_i = tr.make_samples(N, HNu, seed=2)
    coef = tr.schedule_coef(45)
    engines = _rig(N, HNu, P)
    _load(engines, None, Y, Ybar_i, coef)
    for p in _sentinel_positions(N, P):
        r = base.copy(); r[p] = BIG
        _load(engines, r)
        out = _tail(engines, 0.01)
        w = out["w"]
        assert w[p] == f32(1.0) and np.count_nonzero(w) == 1, f"sentinel at {p}: weight {w[p]!r}, {np.count_nonzero(w)} nonzero"
        assert_bit_exact(out["Ybar_im1"][0], tr.update_f32(Y[p], Ybar_i, coef), f"sentinel at {p}: iterate")
    nl = N // P
    # different cluster CTAs, adjacent CTAs, adjacent runs, one run, first/last sample, CTA 7 vs the second wrap of CTA 0,
    # across a rank boundary, first sample of rank 1 vs last of rank 2
    pairs = [(0, 1024), (1023, 1024), (63, 64), (64, 65), (5, N - 1), (7168, 8192), (nl - 1, nl), (nl, 3 * nl - 1)]
    for p, q in pairs:
        if not (0 <= p < q < N):
            continue
        r = base.copy(); r[p] = r[q] = BIG
        _load(engines, r)
        out = _tail(engines, 0.01)
        w = out["w"]
        assert w[p] == f32(0.5) and w[q] == f32(0.5) and np.count_nonzero(w) == 2, f"tie at {p}, {q}: {w[p]!r}, {w[q]!r}"
        ybar = (f32(0.5) * Y[p] + f32(0.5) * Y[q]).astype(f32)
        assert_bit_exact(out["Ybar_im1"][0], tr.update_f32(ybar, Ybar_i, coef), f"tie at {p}, {q}: iterate")


# ---- the column cap ------------------------------------------------------------------------------------------------------

def test_tail_rejects_more_than_27_column_blocks():
    e = _rig(64, 6913, 1)[0]
    L = _lib.lib()
    for fn in (L.mbd_step_tail_launch, L.mbd_step_launch):
        assert fn(e._plan_c, ops._stream()) == -1                    # MBD_EINVAL
        assert b"27 * 256" in L.mbd_last_error()
    torch.cuda.synchronize()
    assert int(e.ctl[2].item()) == 0


# ---- round-1 kernels (MPPI / CMA-ES / CEM statistics) -------------------------------------------------------------------

@pytest.mark.parametrize("N", [1, 1023, 1024, 1025, 2049, 4097, 65536])
def test_round1_kernels_within_f64_bounds(N):
    HNu = 64 if N < 65536 else 8
    Y, Ybar_i = tr.make_samples(N, HNu, seed=3)
    mu = (Ybar_i * f32(0.5)).astype(f32)
    coef = tr.schedule_coef(70)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
    Yd, mud, Ybd = t(Y), t(mu), t(Ybar_i)
    nruns = (N + 63) // 64
    scratch = torch.empty(nruns * HNu, device=DEV)
    for fam in tr.FAMILIES:
        f = tr.make_family(fam, N, tie=(5, N - 1))
        if fam.startswith("demo") and N == 1:
            continue
        for temp in TEMPS:
            what = f"{fam} N={N} temp={temp}"
            ref = tr.reference(f["rews"], temp, f["logpd"], f["rew_xref"], Y, Ybar_i, coef, mu=mu)
            rd, pdd = t(f["rews"]), (None if f["logpd"] is None else t(f["logpd"]))
            w = torch.empty(N, device=DEV); sc = torch.zeros(4, device=DEV); lg = torch.empty(N, device=DEV)
            ops.softmax_weights(rd, pdd, 0, N, temp, f["rew_xref"], w, sc, lg)
            # a slice of the same weights (n_begin != 0: what a rank of a sharded path-integral run asks for)
            nb, nl = N // 3, max(N - N // 3 - 1, 1)
            ws = torch.empty(nl, device=DEV); sc2 = torch.zeros(4, device=DEV)
            ops.softmax_weights(rd, pdd, nb, nl, temp, f["rew_xref"], ws, sc2, lg)
            part = torch.empty(HNu, device=DEV); sq = torch.empty(HNu, device=DEV); out = torch.empty(HNu, device=DEV)
            ops.weighted_sum(w, Yd, HNu, scratch, part)
            ops.weighted_sqerr_sum(w, Yd, mud, HNu, scratch, sq)
            ops.update(part, 1, HNu, Ybd, coef, out)
            torch.cuda.synchronize()
            s = sc.cpu().numpy()
            tr.check_stats(ref, f["rews"], s[0], s[1], tr.cta_depth(N), what)
            if f["logpd"] is not None:
                tr.prepare_demo_terms(ref, f["rews"], f["logpd"], f["rew_xref"], s[0])
            wb = tr.weight_bounds(ref, tr.cta_depth(N), s[0], s[1])
            wh = w.cpu().numpy()
            tr.check_weights(ref, wh, wb, what + ": weights")
            assert_bit_exact(ws.cpu().numpy(), wh[nb:nb + nl], what + ": weights of the slice [n_begin, n_begin + n_local)")
            k = tr.wsum_depth(nruns)
            beta = tr.ybar_bound(ref, Y, wb["rho"], k)
            tr.check_columns(part.cpu().numpy(), ref["Ybar"], beta, what + ": MPPI mean")
            tr.check_columns(sq.cpu().numpy(), ref["sqerr"], tr.sqerr_bound(ref, Y, mu, wb["rho"], k), what + ": CMA-ES spread")
            tr.check_columns(out.cpu().numpy(), ref["Ybar_im1"], tr.update_bound(ref["Ybar"], Ybar_i, coef, beta),
                             what + ": update")


# ---- the step counter stops at step 1 ------------------------------------------------------------------------------------

@pytest.mark.parametrize("graph", [False, True], ids=["direct", "graph-replay"])
def test_step_past_the_end_writes_nothing(graph):
    """One step more than the solve has: the counter is at 0, so the tail would write Ybars[-1] and rew_hist[0].  The
    iterate table is placed at row 1 of a larger tensor whose row 0 is a canary, so even an unguarded kernel writes only
    memory this test owns; the guarded kernels write nothing and report err 2."""
    car = mbd_b200.envs.get_env("car2d")
    Nd, H = 4, 8
    e = eng.DiffusionEngine(car, 128, H, 0.1, False, car.reset(None), Ndiffuse=Nd)
    buf = torch.zeros((Nd + 1, e.HNu), device=DEV)
    buf[0].fill_(123.25)
    e.Ybars = buf[1:]
    e._plan_c = e._make_plan()
    _, alphas, alphas_bar, sigmas = eng.make_schedule(1e-4, 1e-2, Nd)
    e.load_schedule(eng.key_chain(np.uint32([3, 1]), Nd), sigmas, alphas, alphas_bar)
    e.set_step(Nd - 1)
    if graph:
        e.capture()
    for _ in range(Nd - 1):
        e.step()
    torch.cuda.synchronize()
    assert int(e.ctl[0].item()) == 0 and int(e.ctl[2].item()) == 0
    e.check_exchange()
    ybars, hist = e.Ybars.cpu().numpy().copy(), e.rew_hist.cpu().numpy().copy()
    assert np.isfinite(ybars).all()
    e.step()                                              # one too many
    torch.cuda.synchronize()
    assert (buf[0].cpu().numpy() == f32(123.25)).all(), "a step past the end wrote before the iterate table"
    assert_bit_exact(e.Ybars.cpu().numpy(), ybars, "iterates after the extra step")
    assert_bit_exact(e.rew_hist.cpu().numpy(), hist, "reward history after the extra step")
    assert int(e.ctl[0].item()) == 0 and int(e.ctl[2].item()) == 2
    with pytest.raises(ops.MbdError, match="ran past step 1"):
        e.check_exchange()
