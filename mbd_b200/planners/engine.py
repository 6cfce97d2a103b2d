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
import dataclasses
import os
from typing import Optional

import numpy as np
import torch

from .. import _lib, ops, prng
from .sharding import ShardPlan

try:  # tqdm is cosmetic
    from tqdm import tqdm
except Exception:  # noqa: BLE001
    tqdm = None


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


@dataclasses.dataclass(frozen=True)
class LaunchInputs:
    """What launch (1) of a step reads besides the step buffers, on the device: the model blob of a Brax-positional env (None
    for car2d / pushT, whose table is params_car), the initial state (one per problem of a batch), the demonstration (None
    without a demo) and its reward offset, and env_kind, which picks the flat-state env when there is no model.

    `none()` is the form of an engine whose launch (1) reads no env: the black-box objective, MNIST, and engines that drive
    launches 2 and 3 on constructed inputs.  Launch (2) blends the demo in whenever xref is set and reads nothing else of it,
    so such an engine runs a demo tail with any placeholder xref."""
    model: Optional[object] = None
    params_car: Optional[torch.Tensor] = None
    state_init: Optional[torch.Tensor] = None
    xref: Optional[torch.Tensor] = None
    rew_xref: float = 0.0
    env_kind: int = _lib.ENV_CAR2D

    @classmethod
    def none(cls) -> "LaunchInputs":
        return cls()

    @classmethod
    def of_env(cls, env, state_init, enable_demo: bool, d: torch.device, batch: bool = False) -> "LaunchInputs":
        """the inputs of env on device d from one initial state, or with batch from a list of them (state_init [B, state]; the
        problems share the tables and the demonstration).  xref is the demonstration when enable_demo is set."""
        if batch:
            per = [cls.of_env(env, s, enable_demo, d) for s in state_init]
            return dataclasses.replace(per[0], state_init=torch.stack([p.state_init for p in per]).contiguous())
        if env.kind == "pusht" and enable_demo:
            raise ValueError("pushT has no demonstration (mbd_planner.py:118 applies to humanoidtrack / car2d)")
        if env.kind not in ("xpbd", "car2d", "pusht"):
            raise ValueError(env.kind)
        if hasattr(state_init, "pipeline_state"):
            state_init = state_init.pipeline_state if env.kind == "car2d" else state_init.pipeline_state.raw
        x0 = torch.as_tensor(np.ascontiguousarray(state_init, dtype=np.float32), device=d)
        rew_xref = float(getattr(env, "rew_xref", 0.0))
        if env.kind == "xpbd":
            xref = torch.as_tensor(env.xref, device=d).contiguous() if enable_demo else None
            return cls(env.device_model(d), None, x0, xref, rew_xref)
        if env.kind == "car2d":
            params_car, xref = env.device_params()
            return cls(None, params_car, x0, xref if enable_demo else None, rew_xref)
        return cls(None, env.device_params(), x0, None, rew_xref, _lib.ENV_PUSHT)


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




def _device(device) -> torch.device:
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


class StepEngine:
    """The device buffers and the C plan of a three-launch step, and the solve-level API on them.  One solve (B None) or B
    independent solves stepped in lockstep (B >= 1), whose every per-problem buffer is [B, ...] with problem b's single-solve
    block at index b.  A subclass says how a step is launched (`_launch`) and adds the fields of its own to the plan.  P and rank
    are those of a sharded DiffusionEngine rank.

    temp: the plan's temperature; temps: a batch's per-problem temperatures (a [B] device tensor the batched launches read in
    its place).  n_begin / n_local: the samples of this rank (all N by default).  exchange: (rews, logpd, partial) of a sharded
    rank, slices of the buffer its peers read; rews_all / logpd_all then gather every rank's samples."""

    P, rank, group = 1, 0, None

    def __init__(self, inputs: LaunchInputs, N: int, H: int, Nu: int, Ndiffuse: int, enable_demo: bool, B: Optional[int] = None,
                 temp: float = 0.0, temps=None, device: Optional[torch.device] = None, n_begin: int = 0,
                 n_local: Optional[int] = None, exchange=None):
        self.N, self.H, self.Nu, self.Nd, self.B = int(N), int(H), int(Nu), int(Ndiffuse), B
        if self.Nd < 2:
            raise ValueError("Ndiffuse must be at least 2")
        self.HNu = self.H * self.Nu
        self.enable_demo, self.temp = bool(enable_demo), float(temp)
        self.n_begin, self.n_local = int(n_begin), self.N if n_local is None else int(n_local)
        self.device = d = _device(device)
        self.model, self.params_car, self.state_init, self.xref = inputs.model, inputs.params_car, inputs.state_init, inputs.xref
        self.rew_xref, self.env_kind = inputs.rew_xref, inputs.env_kind
        f = dict(device=d, dtype=torch.float32)
        lead, nl, HNu = (() if B is None else (B,)), self.n_local, self.HNu
        self.temps = None if temps is None else torch.tensor(np.asarray(temps, np.float32), device=d)
        self.Y0s = torch.empty(lead + (nl, HNu), **f)
        if exchange is None:
            self.rews = torch.empty(lead + (nl,), **f)
            self.logpd = torch.empty(lead + (nl,), **f) if self.enable_demo else None
            self.partial = torch.empty(HNu, **f)                 # read by sharded steps only; the plan requires it
            self.rews_all, self.logpd_all = self.rews, self.logpd
        else:
            self.rews, self.logpd, self.partial = exchange
            self.rews_all = torch.empty(self.N, **f)
            self.logpd_all = torch.empty(self.N, **f) if self.enable_demo else None
        self.logp_scratch = torch.empty(lead + (self.N,), **f)
        self.weights = torch.empty(lead + (nl,), **f)
        self.scalars = torch.zeros(lead + (4,), **f)
        self.run_scratch = torch.empty(lead + ((nl + ops.RUN - 1) // ops.RUN, HNu), **f)
        # ---- device-resident solve state
        self.Ybars = torch.zeros(lead + (self.Nd, HNu), **f)     # row i = input of step i, row i-1 = its output (row Nd-1 = YN = 0)
        self.rew_hist = torch.zeros(lead + (self.Nd,), **f)      # rews.mean() of step i
        self.params = torch.zeros(lead + (self.Nd, _lib.STEP_PARAMS_WORDS), device=d, dtype=torch.int32)
        self.ctl = torch.zeros(lead + (_lib.STEP_CTL_WORDS,), device=d, dtype=torch.int32)
        self.graph = None
        self._plan_c = self._make_plan()

    # ---- C-ABI plan ----------------------------------------------------------------------------------------------
    def _make_plan(self) -> "_lib.StepPlan":
        p = _lib.StepPlan()
        vp = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        p.model = self.model._h if self.model is not None else None
        p.car_params_dev, p.state_init_dev, p.env_kind = vp(self.params_car), vp(self.state_init), self.env_kind
        p.xref_dev, p.rew_xref = vp(self.xref), self.rew_xref
        p.href = 0 if self.xref is None else int(self.xref.shape[-2])   # xref [href, 2] (car2d) or [ntrack, href, 3] (xpbd)
        p.params_dev, p.ctl_dev, p.Ybars_dev, p.rew_hist_dev = vp(self.params), vp(self.ctl), vp(self.Ybars), vp(self.rew_hist)
        p.n_total, p.n_begin, p.n_local, p.H, p.nu = self.N, self.n_begin, self.n_local, self.H, self.Nu
        p.temp = self.temp
        p.Y0s_dev, p.rews_dev, p.logpd_dev = vp(self.Y0s), vp(self.rews), vp(self.logpd)
        p.rews_all_dev, p.logpd_all_dev, p.logp_dev = vp(self.rews_all), vp(self.logpd_all), vp(self.logp_scratch)
        p.weights_dev, p.runs_dev, p.partial_dev, p.scalars_dev = vp(self.weights), vp(self.run_scratch), vp(self.partial), vp(self.scalars)
        p.P, p.rank = self.P, self.rank
        return p

    # ---- solve-level API -----------------------------------------------------------------------------------------
    def set_step(self, i: int):
        """device step counter <- i, of every problem (the next `step()` runs diffusion step i: reads Ybars[i], writes Ybars[i-1])"""
        self.ctl[..., 0].fill_(int(i))

    def _launch(self):
        """the launches of one step"""
        raise NotImplementedError

    def step(self):
        """one diffusion step at the device-resident step index (the launches, or one replay of the captured graph)"""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._launch()

    def capture(self):
        """records one step in a CUDA graph; later `step()` calls replay it (parameters come from device memory)"""
        i0 = self.ctl[..., 0].clone()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._launch()                       # warm-up outside capture (module load, func attributes)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        if self.P > 1:
            import torch.distributed as dist
            dist.barrier(group=self.group)       # every rank finished its warm-up step before anybody re-arms the counter
        self.ctl[..., 0].copy_(i0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._launch()
        self.graph = g
        return g

    def check_exchange(self):
        """Raises if the device reported an error (`mbd_step_ctl.err`; a batch names its problems): a step ran with the step
        counter already at 0 (one `step()` or graph replay too many; the tail kernels then write nothing), or a cross-GPU
        rendezvous timed out (a peer died or diverged; the outputs are NaN-poisoned).  Synchronises: call it outside the step loop."""
        err = self.ctl[..., 2].cpu().numpy().reshape(-1)
        bad = [int(b) for b in np.nonzero(err)[0]]
        if not bad:
            return
        who = "" if self.B is None else f"problems {bad}: "
        if all(int(err[b]) == 2 for b in bad):
            raise ops.MbdError(f"{who}the step counter ran past step 1 (a step was launched after the last one of the solve); "
                               "that step wrote nothing")
        if self.B is None:
            raise ops.MbdError("cross-GPU rendezvous timed out (a peer rank stopped participating); outputs are NaN")
        raise ops.MbdError(f"{who}device error codes {[int(err[b]) for b in bad]}")

    def solve(self, log=None, log_every: int = 10, desc: Optional[str] = None):
        """Runs a loaded solve: steps Nd - 1 ... 1, one step captured in a CUDA graph and replayed (launched directly under
        MBD_GRAPH=0), then `check_exchange`.  log(i) runs after step i at every log_every-th step and after step 1.  desc: a tqdm
        progress bar with this description, whose postfix is what log returns (without tqdm there is no bar and no log)."""
        self.set_step(self.Nd - 1)
        if os.environ.get("MBD_GRAPH", "1") != "0":
            self.capture()
        steps = range(self.Nd - 1, 0, -1)
        bar = tqdm(steps, desc=desc) if desc is not None and tqdm is not None else None
        if desc is not None and bar is None:
            log = None
        for n_done, i in enumerate(steps if bar is None else bar):
            self.step()
            if log is not None and (n_done % log_every == log_every - 1 or i == 1):
                post = log(i)
                if bar is not None:
                    bar.set_postfix(post)
        self.check_exchange()


class DiffusionEngine(StepEngine):
    def __init__(self, env, Nsample: int, Hsample: int, temp_sample: float, enable_demo: bool, state_init,
                 device: Optional[torch.device] = None, group=None, Ndiffuse: int = 2, emulate=None,
                 inputs: Optional[LaunchInputs] = None, nu: Optional[int] = None):
        """emulate = (P, rank, bufs): rank `rank` of P ranks that all live on THIS device and exchange through the plain
        device buffers `bufs` (one per rank) — the same kernels, flags and peer loads as a real sharded run, used by the
        single-GPU tests (`make_emulated_ranks`).
        env None: an engine of action size nu whose launch (1) reads `inputs` instead of an env's (LaunchInputs.none() for one
        that drives launches 2 and 3 on constructed inputs); state_init is then unused."""
        d = _device(device)
        N, H = int(Nsample), int(Hsample)
        if env is not None:
            inputs, nu = LaunchInputs.of_env(env, state_init, enable_demo, d), env.action_size
        self.plan = ShardPlan.from_env(N, group) if emulate is None else ShardPlan(N, emulate[0], emulate[1], None)
        self.group, self.P, self.rank = group, self.plan.P, self.plan.rank
        nl, HNu = self.plan.n_local, H * nu
        # ---- exchange: P > 1 needs ONE peer-mapped symmetric buffer per rank, [rews n_local | logpd n_local | partial HNu |
        #      2 flag rows of 8 words]; the tail kernels read the peers' slices over NVLink themselves.
        self.sym, self.peer_ptrs = None, None
        self.exchange = "none" if self.P == 1 else "p2p"
        self.off_rews, self.off_logpd, self.off_partial = 0, nl, 2 * nl
        self.off_flags = 2 * nl + HNu
        if self.P > 1 and emulate is not None:
            self.exchange = "p2p-emulated"
            self.sym = emulate[2][self.rank]
            assert self.sym.numel() == 2 * nl + HNu + 16 and self.sym.device == d
            self.peer_ptrs = (ctypes.c_uint64 * self.P)(*[int(b.data_ptr()) for b in emulate[2]])
        elif self.P > 1:
            import torch.distributed as dist
            import torch.distributed._symmetric_memory as symm_mem
            self.sym = symm_mem.empty(2 * nl + HNu + 16, dtype=torch.float32, device=d)
            self.sym.zero_()
            self.sym_hdl = symm_mem.rendezvous(self.sym, dist.group.WORLD if group is None else group)
            self.peer_ptrs = (ctypes.c_uint64 * self.P)(*[int(p) for p in self.sym_hdl.buffer_ptrs])
            torch.cuda.synchronize()
            dist.barrier(group=group)
        exchange = None
        if self.P > 1:
            logpd = self.sym[self.off_logpd:self.off_logpd + nl] if enable_demo else None
            exchange = (self.sym[self.off_rews:self.off_rews + nl], logpd, self.sym[self.off_partial:self.off_partial + HNu])
        super().__init__(inputs, N, H, nu, max(int(Ndiffuse), 2), enable_demo, temp=temp_sample, device=d,
                         n_begin=self.plan.n_begin, n_local=nl, exchange=exchange)
        self.rews_local, self.logpd_local = self.rews, self.logpd   # this rank's samples

    def _make_plan(self) -> "_lib.StepPlan":
        p = super()._make_plan()
        if self.peer_ptrs is not None:
            p.peer_base_ptrs = ctypes.cast(self.peer_ptrs, ctypes.POINTER(ctypes.c_uint64))
        p.off_rews_words, p.off_logpd_words, p.off_partial_words, p.off_flags_words = self.off_rews, self.off_logpd, self.off_partial, self.off_flags
        p.timeout_cycles = int(float(os.environ.get("MBD_XCHG_TIMEOUT_S", "20")) * 2.0e9)
        return p

    def _launch(self):
        ops.step_launch(self._plan_c)

    def load_schedule(self, keys: np.ndarray, sigmas: np.ndarray, alphas: np.ndarray, alphas_bar: np.ndarray):
        """uploads the per-step parameters of a whole solve: row i = {Y0s_rng of step i, sigmas[i], update_coef(i)}"""
        Nd = self.Nd
        if len(sigmas) != Nd or keys.shape != (Nd, 2):
            raise ops.MbdError(f"schedule of {len(sigmas)} steps does not match the engine (Ndiffuse={Nd})")
        self.params.copy_(torch.from_numpy(pack_step_params(keys, sigmas, alphas, alphas_bar)))

    @classmethod
    def make_emulated_ranks(cls, env, Nsample, Hsample, temp_sample, enable_demo, state_init, P: int, Ndiffuse: int = 2, device=None,
                            inputs: Optional[LaunchInputs] = None, nu: Optional[int] = None):
        """P engines = P ranks on ONE device, each with its own stream, exchanging through plain device buffers with the very
        kernels, flags and peer loads of a real sharded run.  Drive them with `step_emulated_ranks`.  env None: see __init__."""
        d = _device(device)
        HNu = int(Hsample) * (env.action_size if env is not None else nu)
        n_local = int(Nsample) // P
        bufs = [torch.zeros(2 * n_local + HNu + 16, device=d) for _ in range(P)]
        engines = [cls(env, Nsample, Hsample, temp_sample, enable_demo, state_init, device=d, Ndiffuse=Ndiffuse, emulate=(P, r, bufs),
                       inputs=inputs, nu=nu) for r in range(P)]
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
        if self.model is not None:
            ops.sample_rollout(self.model, self.state_init, key, self.N, self.n_begin, self.n_local, self.H, float(sigma), Ybar_i,
                               self.Y0s, self.rews_local, xref=self.xref, logpd_out=self.logpd_local)
        elif self.env_kind == _lib.ENV_PUSHT:
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


class BatchedDiffusionEngine(StepEngine):
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
    (DESIGN.md §5m; 1 = the minimum).  0: the mean.  A captured step bakes it in, so it is fixed at construction.

    env None: an engine of action size nu whose launch (1) reads `inputs` (as in DiffusionEngine); state_inits then only count
    the problems."""

    ens_factors: Optional[torch.Tensor] = None   # [B, K, 2] on the device once an ensemble is given
    ens_rews: Optional[torch.Tensor] = None      # [B, N, K]

    def __init__(self, env, Nsample: int, Hsample: int, temps, enable_demo: bool, state_inits, Ndiffuse: int,
                 device: Optional[torch.device] = None, state_buffer: Optional[torch.Tensor] = None, ensemble=None,
                 ens_worst: int = 0, inputs: Optional[LaunchInputs] = None, nu: Optional[int] = None):
        self.env = env
        B = len(state_inits)
        if B < 1 or len(temps) != B:
            raise ValueError(f"{B} initial states and {len(temps)} temperatures: need one of each per problem, B >= 1")
        ens = None if ensemble is None else ensemble_table(ensemble, B, env, enable_demo)
        self.ens_worst = check_ens_worst(ens_worst, None if ens is None else ens.shape[1])
        d = _device(device)
        if env is not None:
            inputs, nu = LaunchInputs.of_env(env, state_inits, enable_demo, d, batch=True), env.action_size
        if state_buffer is not None:
            want = (B, inputs.state_init[0].numel())
            if (not state_buffer.is_cuda or state_buffer.device != d or state_buffer.dtype != torch.float32
                    or not state_buffer.is_contiguous() or tuple(state_buffer.shape) != want):
                raise ValueError(f"state_buffer must be a contiguous float32 tensor of shape {want} on {d} (got "
                                 f"{state_buffer.dtype} {tuple(state_buffer.shape)} on {state_buffer.device})")
            inputs = dataclasses.replace(inputs, state_init=state_buffer)
        if ens is not None:
            self.ens_factors = torch.from_numpy(ens).to(d)
            self.ens_rews = torch.empty((B, int(Nsample), ens.shape[1]), device=d, dtype=torch.float32)
        super().__init__(inputs, Nsample, Hsample, nu, Ndiffuse, enable_demo, B=B, temps=temps, device=d)

    def _make_plan(self) -> "_lib.StepPlan":
        p = super()._make_plan()
        if self.ens_factors is not None:
            p.ens_factors_dev, p.ens_rews_dev, p.ens_k = self.ens_factors.data_ptr(), self.ens_rews.data_ptr(), self.ens_factors.shape[1]
            p.ens_worst = self.ens_worst
        return p

    def set_ensemble(self, table):
        """rewrites the planner ensemble in place (same B and K): a captured step reads the new values on its next replay"""
        if self.ens_factors is None:
            raise ValueError("this engine was built without a planner ensemble")
        ens = ensemble_table(table, self.B, self.env, self.enable_demo)
        if ens.shape != tuple(self.ens_factors.shape):
            raise ValueError(f"the ensemble must keep its shape {tuple(self.ens_factors.shape)} (got {ens.shape})")
        self.ens_factors.copy_(torch.from_numpy(ens))

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

    def _launch(self):
        """the three launches of one step of every problem"""
        ops.batch_step_launch(self._plan_c, self.B, self.Nd, self.temps)

    def problem(self, b: int):
        """the single-problem view of problem b that `final_reward` and the rollout helpers take (model, tables, state_init)"""
        from types import SimpleNamespace
        return SimpleNamespace(model=self.model, params_car=self.params_car, state_init=self.state_init[b], H=self.H, Nu=self.Nu)
