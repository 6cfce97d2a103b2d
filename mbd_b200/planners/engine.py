"""Device-side engine of one reverse-diffusion step (`reverse_once`,
upstream mbd/planners/mbd_planner.py:97-135), sample-sharded over ranks.

A step is THREE launches at any rank count (`mbd_step_launch`, csrc/step_tail.cuh):
  1. fused sampling + rollouts                      -> Y0s_local, rews_local (+logpd_local)
  2. k_step_weights: one 8-CTA cluster; sharded, it rendezvous with the peer GPUs and pulls their per-sample returns
     over NVLink itself, then global mean / std / demo blend / softmax           -> weights_local
  3. k_step_update: weighted-mean runs; the last CTA folds the tree, exchanges the rank partials over NVLink (sharded)
     and applies the update lines 130-133                                         -> Ybars[i - 1], ctl.i -= 1
Everything that changes from step to step (PRNG key, sigma, schedule scalars, the step index, the iterate) lives in DEVICE
memory, so the three launches take no per-step host arguments: `load_schedule` uploads the whole solve once, `capture`
records one step in a CUDA graph and `step` replays it — the host loop of mbd_planner.py:138-148 no longer bounds a solve.
Rank r of P owns samples [r*N/P, (r+1)*N/P); noise is addressed by GLOBAL index, all reduction orders depend on N only,
so the result does not depend on P.  Sharded runs need torch symmetric memory (NVLink peer access); there is no NCCL call
on the path (NCCL only bootstraps the rendezvous of the symmetric buffer).
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import numpy as np
import torch

from .. import _lib, ops, prng
from .sharding import ShardPlan


def linspace_f32(start: float, stop: float, num: int) -> np.ndarray:
    """`jnp.linspace(start, stop, num)` with x64 disabled (mbd_planner.py:13-14 leaves it off) **[jax-recalled]**: JAX does not
    compute `start + k * delta`; it blends the endpoints in float32, `start * (1 - k/(num-1)) + stop * (k/(num-1))`, and appends
    `stop` itself as the last element.  NumPy's float64 formula rounded to float32 differs from this by an ulp in a few entries
    (VERDICT r1, row a2); `MBD_LINSPACE=numpy` restores it."""
    import os
    f = np.float32
    if os.environ.get("MBD_LINSPACE", "jax") == "numpy" or num < 2:
        return np.linspace(start, stop, num, dtype=f)
    div = f(num - 1)
    step = (np.arange(num - 1, dtype=f) / div).astype(f)
    out = (f(start) * (f(1.0) - step)).astype(f) + (f(stop) * step).astype(f)
    return np.concatenate([out.astype(f), np.array([stop], dtype=f)])


def make_schedule(beta0: float, betaT: float, Ndiffuse: int):
    """mbd_planner.py:84-87 in float32."""
    betas = linspace_f32(beta0, betaT, Ndiffuse)
    alphas = (np.float32(1.0) - betas).astype(np.float32)
    alphas_bar = np.cumprod(alphas, dtype=np.float32)
    sigmas = np.sqrt(np.float32(1.0) - alphas_bar).astype(np.float32)
    return betas, alphas, alphas_bar, sigmas


def update_coef(alphas, alphas_bar, i: int):
    """The float32 scalars of mbd_planner.py:100,130-133 for step i."""
    one = np.float32(1.0)
    ab = np.float32(alphas_bar[i])
    return [np.sqrt(ab), one / (one - ab), one - ab, one / np.sqrt(np.float32(alphas[i])), np.sqrt(np.float32(alphas_bar[i - 1]))]


def key_chain(rng_exp, Ndiffuse: int) -> np.ndarray:
    """The Y0s_rng of every step: `rng, Y0s_rng = split(rng)` per step starting from rng_exp (mbd_planner.py:103,150).
    Returns [Ndiffuse, 2] uint32 with row i = key of step i (rows 0 and beyond the chain are zero)."""
    keys = np.zeros((Ndiffuse, 2), np.uint32)
    r = np.asarray(rng_exp, np.uint32)
    for i in range(Ndiffuse - 1, 0, -1):
        r, k = prng.split2(r)
        keys[i] = k
    return keys


def pack_step_params(keys: np.ndarray, sigmas: np.ndarray, alphas: Optional[np.ndarray], alphas_bar: Optional[np.ndarray]) -> np.ndarray:
    """The device table of a whole solve (`mbd_step_params` rows, as int32 words): row i = {Y0s_rng of step i, sigmas[i],
    update_coef(i)}.  Row 0 carries the key and sigma only (step 0 is never run).  alphas None (the path-integral baselines,
    which have no schedule): every coefficient is 0."""
    Nd = len(sigmas)
    if keys.shape != (Nd, 2):
        raise ops.MbdError(f"key chain of shape {keys.shape} does not match a schedule of {Nd} steps")
    tab = np.zeros((Nd, _lib.STEP_PARAMS_WORDS), np.uint32)
    tab[:, 0:2] = keys
    tab[:, 2] = np.asarray(sigmas, np.float32).view(np.uint32)
    for i in range(1, Nd if alphas is not None else 0):
        tab[i, 3:8] = np.asarray(update_coef(alphas, alphas_bar, i), np.float32).view(np.uint32)
    return tab.view(np.int32)


def env_tensors(env, state_init, enable_demo: bool, d: torch.device):
    """(model, params_car, state_init, xref) of one env on device d: what launch (1) of a step reads.  model is the
    device-resident blob of a Brax-positional env (None for car2d / pushT, whose table is params_car); xref is the
    demonstration when enable_demo is set."""
    if env.kind == "xpbd":
        raw = state_init.pipeline_state.raw if hasattr(state_init, "pipeline_state") else state_init
        xref = torch.as_tensor(env.xref, device=d).contiguous() if enable_demo else None
        return env.device_model(d), None, torch.as_tensor(np.ascontiguousarray(raw, dtype=np.float32), device=d), xref
    if env.kind == "car2d":
        params_car, xref = env.device_params()
        x0 = state_init.pipeline_state if hasattr(state_init, "pipeline_state") else state_init
        return None, params_car, torch.as_tensor(np.ascontiguousarray(x0, dtype=np.float32), device=d), (xref if enable_demo else None)
    if env.kind == "pusht":
        if enable_demo:
            raise ValueError("pushT has no demonstration (mbd_planner.py:118 applies to humanoidtrack / car2d)")
        raw = state_init.pipeline_state.raw if hasattr(state_init, "pipeline_state") else state_init
        return None, env.device_params(), torch.as_tensor(np.ascontiguousarray(raw, dtype=np.float32), device=d), None
    raise ValueError(env.kind)


def ensemble_table(table, B: int, env, enable_demo: bool) -> np.ndarray:
    """a planner ensemble as the float32 [B, K, 2] table of mbd_step_plan.ens_factors_dev: table[b][k] = (friction factor, gear
    factor) of member k of problem b, member-major within each problem.  ValueError unless the env is positional (xpbd), there is no
    demo, the shape is [B, K, 2] with 1 <= K <= ENS_MAXK and every value is finite and >= 0 in float32."""
    if getattr(env, "kind", None) != "xpbd":
        raise ValueError(f"planner ensembles exist for the positional (xpbd) envs only, not {type(env).__name__}")
    if enable_demo:
        raise ValueError("a planner ensemble has no demonstration (enable_demo must be False)")
    if isinstance(table, torch.Tensor):
        table = table.detach().cpu().numpy()
    t = np.asarray(table, dtype=np.float64)
    if t.ndim != 3 or t.shape[0] != B or t.shape[2] != 2 or not 1 <= t.shape[1] <= _lib.ENS_MAXK:
        raise ValueError(f"the ensemble must have shape ({B}, K, 2) with 1 <= K <= {_lib.ENS_MAXK} (got {t.shape})")
    with np.errstate(over="ignore"):
        f = np.ascontiguousarray(t.astype(np.float32))
    if not (np.isfinite(f).all() and (f >= 0).all()):
        raise ValueError(f"ensemble factors must be finite and >= 0 (got {t.reshape(-1).tolist()})")
    return f


def check_ens_worst(worst, K: Optional[int]) -> int:
    """mbd_step_plan.ens_worst of an ensemble of K members (None: no ensemble): an int in 0 .. K, and 0 without an ensemble
    (ValueError)"""
    if isinstance(worst, bool) or not isinstance(worst, (int, np.integer)):
        raise ValueError(f"ens_worst must be an int (got {worst!r})")
    if K is None and worst != 0:
        raise ValueError(f"ens_worst = {worst} needs a planner ensemble")
    if K is not None and not 0 <= worst <= K:
        raise ValueError(f"ens_worst must be in 0 .. K = {K} (got {worst})")
    return int(worst)


def xref_len(env, xref) -> int:
    """href of the step plan: the demonstration's length in steps (0 without one)"""
    return 0 if xref is None else int(xref.shape[1] if env.kind == "xpbd" else xref.shape[0])


class DiffusionEngine:
    def __init__(self, env, Nsample: int, Hsample: int, temp_sample: float, enable_demo: bool, state_init,
                 device: Optional[torch.device] = None, group=None, Ndiffuse: int = 2, emulate=None):
        """emulate = (P, rank, bufs): rank `rank` of P ranks that all live on THIS device and exchange through the plain
        device buffers `bufs` (one per rank) — the same kernels, flags and peer loads as a real sharded run, used by the
        single-GPU tests (`make_emulated_ranks`)."""
        self.env = env
        self.N, self.H, self.temp = int(Nsample), int(Hsample), float(temp_sample)
        self.enable_demo = bool(enable_demo)
        self.plan = ShardPlan.from_env(self.N, group) if emulate is None else ShardPlan(self.N, emulate[0], emulate[1], None)
        self.group, self.P, self.rank = group, self.plan.P, self.plan.rank
        self.n_local, self.n_begin = self.plan.n_local, self.plan.n_begin
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.Nu = env.action_size
        self.HNu = self.H * self.Nu
        self.Nd = max(int(Ndiffuse), 2)
        d = self.device
        f = dict(device=d, dtype=torch.float32)
        self.Y0s = torch.empty((self.n_local, self.HNu), **f)
        # ---- exchange: P > 1 needs ONE peer-mapped symmetric buffer per rank, [rews n_local | logpd n_local | partial HNu |
        #      2 flag rows of 8 words]; the tail kernels read the peers' slices over NVLink themselves.
        self.sym, self.peer_ptrs = None, None
        self.exchange = "none" if self.P == 1 else "p2p"
        self.off_rews, self.off_logpd, self.off_partial = 0, self.n_local, 2 * self.n_local
        self.off_flags = 2 * self.n_local + self.HNu
        if self.P > 1 and emulate is not None:
            self.exchange = "p2p-emulated"
            self.sym = emulate[2][self.rank]
            assert self.sym.numel() == 2 * self.n_local + self.HNu + 16 and self.sym.device == d
            self.peer_ptrs = (ctypes.c_uint64 * self.P)(*[int(b.data_ptr()) for b in emulate[2]])
        elif self.P > 1:
            import torch.distributed as dist
            import torch.distributed._symmetric_memory as symm_mem
            words = 2 * self.n_local + self.HNu + 16
            self.sym = symm_mem.empty(words, dtype=torch.float32, device=d)
            self.sym.zero_()
            self.sym_hdl = symm_mem.rendezvous(self.sym, dist.group.WORLD if group is None else group)
            self.peer_ptrs = (ctypes.c_uint64 * self.P)(*[int(p) for p in self.sym_hdl.buffer_ptrs])
            torch.cuda.synchronize()
            dist.barrier(group=group)
        if self.P > 1:
            self.rews_local = self.sym[self.off_rews:self.off_rews + self.n_local]
            self.logpd_local = self.sym[self.off_logpd:self.off_logpd + self.n_local] if self.enable_demo else None
            self.partial = self.sym[self.off_partial:self.off_partial + self.HNu]
            self.rews_all = torch.empty(self.N, **f)
            self.logpd_all = torch.empty(self.N, **f) if self.enable_demo else None
        else:
            self.rews_local = torch.empty(self.n_local, **f)
            self.logpd_local = torch.empty(self.n_local, **f) if self.enable_demo else None
            self.partial = torch.empty(self.HNu, **f)
            self.rews_all, self.logpd_all = self.rews_local, self.logpd_local
        self.weights = torch.empty(self.n_local, **f)
        self.scalars = torch.zeros(4, **f)
        self.logp_scratch = torch.empty(self.N, **f)
        self.run_scratch = torch.empty(((self.n_local + ops.RUN - 1) // ops.RUN) * self.HNu, **f)
        # ---- device-resident solve state
        self.Ybars = torch.zeros((self.Nd, self.HNu), **f)        # row i = input of step i, row i-1 = its output (row Nd-1 = YN = 0)
        self.rew_hist = torch.zeros(self.Nd, **f)                 # rews.mean() of step i
        self.params = torch.zeros((self.Nd, _lib.STEP_PARAMS_WORDS), device=d, dtype=torch.int32)
        self.ctl = torch.zeros(_lib.STEP_CTL_WORDS, device=d, dtype=torch.int32)
        self.launches_per_step = 3
        self.launches_last_step = 3
        self.graph = None
        self.model, self.params_car, self.state_init, self.xref = env_tensors(env, state_init, self.enable_demo, d)
        self.rew_xref = float(getattr(env, "rew_xref", 0.0))
        self._plan_c = self._make_plan()

    # ---- C-ABI plan ----------------------------------------------------------------------------------------------
    def _make_plan(self) -> "_lib.StepPlan":
        p = _lib.StepPlan()
        vp = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        p.model = self.model._h if self.model is not None else None
        p.car_params_dev = vp(self.params_car)
        p.state_init_dev = vp(self.state_init)
        p.params_dev, p.ctl_dev, p.Ybars_dev, p.rew_hist_dev = vp(self.params), vp(self.ctl), vp(self.Ybars), vp(self.rew_hist)
        p.n_total, p.n_begin, p.n_local, p.H, p.nu = self.N, self.n_begin, self.n_local, self.H, self.Nu
        p.temp, p.rew_xref = self.temp, self.rew_xref
        p.xref_dev = vp(self.xref)
        p.env_kind = _lib.ENV_PUSHT if self.env.kind == "pusht" else _lib.ENV_CAR2D
        p.href = xref_len(self.env, self.xref)
        p.Y0s_dev, p.rews_dev, p.logpd_dev = vp(self.Y0s), vp(self.rews_local), vp(self.logpd_local)
        p.rews_all_dev, p.logpd_all_dev, p.logp_dev = vp(self.rews_all), vp(self.logpd_all), vp(self.logp_scratch)
        p.weights_dev, p.runs_dev, p.partial_dev, p.scalars_dev = vp(self.weights), vp(self.run_scratch), vp(self.partial), vp(self.scalars)
        p.P, p.rank = self.P, self.rank
        if self.peer_ptrs is not None:
            p.peer_base_ptrs = ctypes.cast(self.peer_ptrs, ctypes.POINTER(ctypes.c_uint64))
        p.off_rews_words, p.off_logpd_words, p.off_partial_words, p.off_flags_words = self.off_rews, self.off_logpd, self.off_partial, self.off_flags
        p.timeout_cycles = int(float(os.environ.get("MBD_XCHG_TIMEOUT_S", "20")) * 2.0e9)
        return p

    # ---- solve-level API -----------------------------------------------------------------------------------------
    def load_schedule(self, keys: np.ndarray, sigmas: np.ndarray, alphas: np.ndarray, alphas_bar: np.ndarray):
        """uploads the per-step parameters of a whole solve: row i = {Y0s_rng of step i, sigmas[i], update_coef(i)}"""
        Nd = self.Nd
        if len(sigmas) != Nd or keys.shape != (Nd, 2):
            raise ops.MbdError(f"schedule of {len(sigmas)} steps does not match the engine (Ndiffuse={Nd})")
        self.params.copy_(torch.from_numpy(pack_step_params(keys, sigmas, alphas, alphas_bar)))

    def set_step(self, i: int):
        """device step counter <- i (the next `step()` runs diffusion step i: reads Ybars[i], writes Ybars[i-1])"""
        self.ctl[0:1].fill_(int(i))

    def step(self):
        """one diffusion step at the device-resident step index (three launches, or one replay of the captured graph)"""
        if self.graph is not None:
            self.graph.replay()
        else:
            ops.step_launch(self._plan_c)

    def capture(self):
        """records one step in a CUDA graph; later `step()` calls replay it (parameters come from device memory)"""
        i0 = int(self.ctl[0].item())
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.step_launch(self._plan_c)        # warm-up outside capture (module load, func attributes)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        if self.P > 1:
            import torch.distributed as dist
            dist.barrier(group=self.group)       # every rank finished its warm-up step before anybody re-arms the counter
        self.set_step(i0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ops.step_launch(self._plan_c)
        self.graph = g
        return g

    def check_exchange(self):
        """Raises if the device reported an error (`mbd_step_ctl.err`): a cross-GPU rendezvous timed out (a peer died or
        diverged; the outputs are NaN-poisoned), or a step ran with the step counter already at 0 (one `step()` or graph
        replay too many; the tail kernels then write nothing).  Synchronises: call it outside the step loop."""
        err = int(self.ctl[2].item())
        if err == 2:
            raise ops.MbdError("the step counter ran past step 1 (a step was launched after the last one of the solve); "
                               "that step wrote nothing")
        if err != 0:
            raise ops.MbdError("cross-GPU rendezvous timed out (a peer rank stopped participating); outputs are NaN")

    @classmethod
    def make_emulated_ranks(cls, env, Nsample, Hsample, temp_sample, enable_demo, state_init, P: int, Ndiffuse: int = 2, device=None):
        """P engines = P ranks on ONE device, each with its own stream, exchanging through plain device buffers with the very
        kernels, flags and peer loads of a real sharded run.  Drive them with `step_emulated_ranks`."""
        d = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        HNu = int(Hsample) * env.action_size
        n_local = int(Nsample) // P
        bufs = [torch.zeros(2 * n_local + HNu + 16, device=d) for _ in range(P)]
        engines = [cls(env, Nsample, Hsample, temp_sample, enable_demo, state_init, device=d, Ndiffuse=Ndiffuse, emulate=(P, r, bufs))
                   for r in range(P)]
        for e in engines:
            e.stream = torch.cuda.Stream(device=d)
        return engines

    @staticmethod
    def step_emulated_ranks(engines, ranks=None):
        """launches one step of every (or the given) emulated rank on its own stream — they rendezvous on the device"""
        cur = torch.cuda.current_stream()
        for e in engines:
            e.stream.wait_stream(cur)
        for r, e in enumerate(engines):
            if ranks is None or r in ranks:
                with torch.cuda.stream(e.stream):
                    e.step()
        for e in engines:
            cur.wait_stream(e.stream)

    def rollout_phase(self, key, sigma: float, Ybar_i: torch.Tensor):
        """sampling + rollouts with host-side parameters (path_integral.py's update_once shares it)"""
        if self.env.kind == "xpbd":
            ops.sample_rollout(self.model, self.state_init, key, self.N, self.n_begin, self.n_local, self.H, float(sigma), Ybar_i,
                               self.Y0s, self.rews_local, xref=self.xref, logpd_out=self.logpd_local)
        elif self.env.kind == "pusht":
            ops.pusht_rollout(self.params_car, self.state_init, self.Y0s.view(self.n_local, self.H, 2), key=key, n_total=self.N,
                              n_begin=self.n_begin, sigma=float(sigma), Ybar=Ybar_i, rews_out=self.rews_local)
        else:
            ops.car2d_rollout(self.params_car, self.state_init, self.Y0s.view(self.n_local, self.H, 2), xref=self.xref, key=key,
                              n_total=self.N, n_begin=self.n_begin, sigma=float(sigma), Ybar=Ybar_i, rews_out=self.rews_local,
                              logpd_out=self.logpd_local)

    def stage_step(self, key, sigma: float, Ybar_i: torch.Tensor, coef, i: int = 1):
        """host-side parameters of ONE step -> row i of the device tables; the next `step()` runs it"""
        row = np.zeros(_lib.STEP_PARAMS_WORDS, np.uint32)
        row[0:2] = np.asarray(key, np.uint32)
        row[2] = np.float32(sigma).view(np.uint32)
        row[3:8] = np.asarray(coef, np.float32).view(np.uint32)
        self.params[i].copy_(torch.from_numpy(row.view(np.int32)))
        self.Ybars[i].copy_(Ybar_i)
        self.set_step(i)

    # ---- single-step API (tests, bench, path-compatible with round 1) ---------------------------------------------
    def reverse_once(self, key, sigma: float, Ybar_i: torch.Tensor, coef, out: Optional[torch.Tensor] = None):
        """One diffusion step with host-side parameters: stages them into row 1 of the device tables, runs the step,
        returns (Ybar_im1 [HNu] device tensor, rews.mean() device scalar view)."""
        self.stage_step(key, sigma, Ybar_i, coef, 1)
        g, self.graph = self.graph, None
        try:
            self.step()
        finally:
            self.graph = g
        res = self.Ybars[0]
        if out is not None:
            out.copy_(res)
            res = out
        return res, self.scalars[0]


class BatchedDiffusionEngine:
    """B independent solves of one env and shape (N, H, Ndiffuse, demo) stepped in lockstep: ONE three-launch step
    (`mbd_batch_step_launch`) advances all of them.  Problem b has its own initial state, key chain, schedule (beta0 / betaT
    may differ) and temperature; every per-problem device buffer is [B, ...] with problem b's single-solve block at index b.
    The noise of problem b is drawn from its own key with problem-local counters and every reduction order depends on N only,
    so problem b reproduces the `DiffusionEngine` solve of the same inputs bit for bit.  One GPU (P = 1).

    state_buffer: an external [B, S] float32 device tensor the steps read the initial states from instead of the engine's own copy
    of `state_inits` (the receding-horizon controller passes `VecEnv.state`, so every step plans from the plant's current state).
    Its layout must be the engine's; its content is the caller's (`state_inits` then only fix the layout).

    ensemble: a planner ensemble [B][K][2] (DESIGN.md §5l, positional envs, no demo): problem b rolls every sample out under the K
    models (friction ensemble[b][k][0], gear ensemble[b][k][1]) and the tail reads the mean of the K returns.  `ens_rews` [B, N, K]
    holds every member return of the last step.  None: today's step.

    ens_worst: with an ensemble, m in 1 .. K scores every sample by the mean of its m worst member returns instead of all K
    (DESIGN.md §5m; 1 = the minimum).  0: the mean.  A captured step bakes it in, so it is fixed at construction."""

    ens_factors: Optional[torch.Tensor] = None   # [B, K, 2] on the device once an ensemble is given
    ens_rews: Optional[torch.Tensor] = None      # [B, N, K]

    def __init__(self, env, Nsample: int, Hsample: int, temps, enable_demo: bool, state_inits, Ndiffuse: int,
                 device: Optional[torch.device] = None, state_buffer: Optional[torch.Tensor] = None, ensemble=None,
                 ens_worst: int = 0):
        self.env = env
        self.B = len(state_inits)
        if self.B < 1 or len(temps) != self.B:
            raise ValueError(f"{self.B} initial states and {len(temps)} temperatures: need one of each per problem, B >= 1")
        ens = None if ensemble is None else ensemble_table(ensemble, self.B, env, enable_demo)
        self.ens_worst = check_ens_worst(ens_worst, None if ens is None else ens.shape[1])
        self.N, self.H = int(Nsample), int(Hsample)
        self.enable_demo = bool(enable_demo)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.Nu = env.action_size
        self.HNu = self.H * self.Nu
        self.Nd = int(Ndiffuse)
        if self.Nd < 2:
            raise ValueError("Ndiffuse must be at least 2")
        per = [env_tensors(env, s, self.enable_demo, self.device) for s in state_inits]
        self.model, self.params_car, _, self.xref = per[0]              # shared by every problem
        self.state_init = torch.stack([p[2] for p in per]).contiguous()  # [B, state]
        if state_buffer is not None:
            want = (self.B, self.state_init[0].numel())
            if (not state_buffer.is_cuda or state_buffer.device != self.device or state_buffer.dtype != torch.float32
                    or not state_buffer.is_contiguous() or tuple(state_buffer.shape) != want):
                raise ValueError(f"state_buffer must be a contiguous float32 tensor of shape {want} on {self.device} (got "
                                 f"{state_buffer.dtype} {tuple(state_buffer.shape)} on {state_buffer.device})")
            self.state_init = state_buffer
        self.rew_xref = float(getattr(env, "rew_xref", 0.0))
        self._alloc(temps)
        if ens is not None:
            K = ens.shape[1]
            self.ens_factors = torch.from_numpy(ens).to(self.device)
            self.ens_rews = torch.empty((self.B, self.N, K), device=self.device, dtype=torch.float32)
            p = self._plan_c
            p.ens_factors_dev, p.ens_rews_dev, p.ens_k = self.ens_factors.data_ptr(), self.ens_rews.data_ptr(), K
            p.ens_worst = self.ens_worst

    def set_ensemble(self, table):
        """rewrites the planner ensemble in place (same B and K): a captured step reads the new values on its next replay"""
        if self.ens_factors is None:
            raise ValueError("this engine was built without a planner ensemble")
        ens = ensemble_table(table, self.B, self.env, self.enable_demo)
        if ens.shape != tuple(self.ens_factors.shape):
            raise ValueError(f"the ensemble must keep its shape {tuple(self.ens_factors.shape)} (got {ens.shape})")
        self.ens_factors.copy_(torch.from_numpy(ens))

    def _alloc(self, temps):
        """the per-problem device buffers and the C plan, from B, N, HNu, Nd, enable_demo and the env tensors set before"""
        B, N, d = self.B, self.N, self.device
        f = dict(device=d, dtype=torch.float32)
        self.temps = torch.tensor(np.asarray(temps, np.float32), device=d)
        self.Y0s = torch.empty((B, N, self.HNu), **f)
        self.rews = torch.empty((B, N), **f)
        self.logpd = torch.empty((B, N), **f) if self.enable_demo else None
        self.logp_scratch = torch.empty((B, N), **f)
        self.weights = torch.empty((B, N), **f)
        self.scalars = torch.zeros((B, 4), **f)
        self.run_scratch = torch.empty((B, (N + ops.RUN - 1) // ops.RUN, self.HNu), **f)
        self.partial = torch.empty(self.HNu, **f)                       # read by sharded steps only; the plan requires it
        self.Ybars = torch.zeros((B, self.Nd, self.HNu), **f)
        self.rew_hist = torch.zeros((B, self.Nd), **f)
        self.params = torch.zeros((B, self.Nd, _lib.STEP_PARAMS_WORDS), device=d, dtype=torch.int32)
        self.ctl = torch.zeros((B, _lib.STEP_CTL_WORDS), device=d, dtype=torch.int32)
        self.graph = None
        self._plan_c = self._make_plan()

    def _make_plan(self) -> "_lib.StepPlan":
        p = _lib.StepPlan()
        vp = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        p.model = self.model._h if self.model is not None else None
        p.car_params_dev, p.state_init_dev = vp(self.params_car), vp(self.state_init)
        p.params_dev, p.ctl_dev, p.Ybars_dev, p.rew_hist_dev = vp(self.params), vp(self.ctl), vp(self.Ybars), vp(self.rew_hist)
        p.n_total, p.n_begin, p.n_local, p.H, p.nu = self.N, 0, self.N, self.H, self.Nu
        p.temp, p.rew_xref = 0.0, self.rew_xref      # the per-problem temperatures come from self.temps
        p.xref_dev = vp(self.xref)
        p.env_kind = _lib.ENV_PUSHT if self.env.kind == "pusht" else _lib.ENV_CAR2D
        p.href = xref_len(self.env, self.xref)
        p.Y0s_dev, p.rews_dev, p.logpd_dev = vp(self.Y0s), vp(self.rews), vp(self.logpd)
        p.rews_all_dev, p.logpd_all_dev, p.logp_dev = vp(self.rews), vp(self.logpd), vp(self.logp_scratch)
        p.weights_dev, p.runs_dev, p.partial_dev, p.scalars_dev = vp(self.weights), vp(self.run_scratch), vp(self.partial), vp(self.scalars)
        p.P, p.rank = 1, 0
        return p

    # ---- solve-level API (that of DiffusionEngine, one entry per problem) -----------------------------------------------
    def load_schedule(self, keys, sigmas, alphas, alphas_bar):
        """uploads every problem's solve: keys[b] [Ndiffuse, 2] (key_chain), sigmas[b] / alphas[b] / alphas_bar[b] (make_schedule)"""
        if not (len(keys) == len(sigmas) == len(alphas) == len(alphas_bar) == self.B):
            raise ops.MbdError(f"need {self.B} key chains and schedules, one per problem")
        for b in range(self.B):
            if len(sigmas[b]) != self.Nd:
                raise ops.MbdError(f"problem {b}: schedule of {len(sigmas[b])} steps does not match the engine (Ndiffuse={self.Nd})")
        tab = np.stack([pack_step_params(np.asarray(keys[b]), sigmas[b], alphas[b], alphas_bar[b]) for b in range(self.B)])
        self.params.copy_(torch.from_numpy(tab))

    def set_step(self, i: int):
        """every problem's device step counter <- i"""
        self.ctl[:, 0].fill_(int(i))

    def step(self):
        """one diffusion step of every problem (three launches, or one replay of the captured graph)"""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._launch()

    def _launch(self):
        """the three launches of one step of every problem"""
        ops.batch_step_launch(self._plan_c, self.B, self.Nd, self.temps)

    def capture(self):
        """records one batched step in a CUDA graph; later `step()` calls replay it"""
        i0 = self.ctl[:, 0].clone()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._launch()   # warm-up outside capture
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.ctl[:, 0].copy_(i0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._launch()
        self.graph = g
        return g

    def check_exchange(self):
        """Raises if any problem's control block reports an error, naming the problems: err 2 = a step ran with the step
        counter already at 0 (one `step()` or replay too many; that step wrote nothing).  Synchronises."""
        err = self.ctl[:, 2].cpu().numpy()
        bad = [int(b) for b in np.nonzero(err)[0]]
        if not bad:
            return
        if all(int(err[b]) == 2 for b in bad):
            raise ops.MbdError(f"problems {bad}: the step counter ran past step 1 (a step was launched after the last one of "
                               "the solve); that step wrote nothing")
        raise ops.MbdError(f"problems {bad}: device error codes {[int(err[b]) for b in bad]}")

    def problem(self, b: int):
        """the single-problem view of problem b that `final_reward` and the rollout helpers take (model, tables, state_init)"""
        from types import SimpleNamespace
        return SimpleNamespace(model=self.model, params_car=self.params_car, state_init=self.state_init[b], H=self.H, Nu=self.Nu)
