"""Torch-tensor front end of the C ABI (include/mbd_b200.h).

PyTorch is plumbing here: it owns device memory and the CUDA stream; every compute call goes
through ctypes into libmbd_b200.so with raw device pointers.  There is no CPU/eager fallback:
all functions raise `MbdError` without a CUDA device.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._lib import MbdError, check, key_ptr

RUN = 64  # samples per sequential run in mbd_weighted_sum (kRun in csrc/mbd_b200.cu)


def _p(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(t: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    if not t.is_cuda:
        raise MbdError("expected a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype or not t.is_contiguous():
        raise MbdError(f"expected a contiguous {dtype} tensor, got {t.dtype} contiguous={t.is_contiguous()}")
    return t


def set_kernel_variant(v: int):
    """0 = auto, 1 = lane-per-link kernel, 2/3 = warp-per-link kernel with CTA / named-barrier sync,
    8 = packed kernel, two samples per lane (all bit-identical; 3 and 8 fall back to 2 on models they do not cover)."""
    check(_lib.lib().mbd_set_kernel_variant(int(v)), "mbd_set_kernel_variant")


class Model:
    """Device-resident compiled model (mbd_model_create)."""

    def __init__(self, blob: np.ndarray, device: Optional[torch.device] = None):
        _lib.require_gpu()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        blob = np.ascontiguousarray(blob, dtype=np.uint32)
        self.blob = blob
        hdr = blob.view(np.int32)
        self.L, self.nu, self.n_frames, self.reward, self.ntrack = (int(hdr[i]) for i in range(1, 6))
        with torch.cuda.device(self.device):
            self._h = _lib.lib().mbd_model_create(blob.ctypes.data_as(_lib.c_u32p), blob.size)
        if not self._h:
            raise MbdError("mbd_model_create failed: " + _lib.lib().mbd_last_error().decode())

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.lib().mbd_model_destroy(ctypes.c_void_p(h))
            except Exception:  # noqa: BLE001  (interpreter shutdown)
                pass

    @property
    def handle(self):
        return ctypes.c_void_p(self._h)


def sample(key, n_total: int, n_begin: int, n_local: int, HNu: int, sigma: float, Ybar: torch.Tensor,
           out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _lib.require_gpu()
    Ybar = _dev(Ybar)
    out = torch.empty((n_local, HNu), device=Ybar.device, dtype=torch.float32) if out is None else _dev(out)
    k, kp = key_ptr(key)
    check(_lib.lib().mbd_sample(kp, n_total, n_begin, n_local, HNu, ctypes.c_float(sigma), _p(Ybar), _p(out), _stream()), "mbd_sample")
    return out


def rollout(model: Model, state_init: torch.Tensor, Y0s: torch.Tensor, xref: Optional[torch.Tensor] = None,
            want_rewss=False, want_final=False, want_track=False, nsub_override: int = 0, want_traj=False):
    """vmap(rollout_us)(state_init, Y0s): Y0s [n,H,nu] -> dict(rews [n], rewss, logpd, final, track, traj).
    want_traj: traj [n,H,L,13], every link's raw state after each step (mbd_rollout_traj, the warp-per-link kernel)."""
    state_init, Y0s = _dev(state_init), _dev(Y0s)
    n, H, nu = Y0s.shape
    if nu != model.nu or state_init.numel() != model.L * 13:
        raise MbdError("shape mismatch between model, state_init and Y0s")
    dev = Y0s.device
    rews = torch.empty(n, device=dev)
    rewss = torch.empty((n, H), device=dev) if want_rewss else None
    final = torch.empty((n, model.L, 13), device=dev) if want_final else None
    track = torch.empty((n, H, model.ntrack, 3), device=dev) if want_track else None
    logpd, href = None, 0
    if xref is not None:
        xref = _dev(xref)
        href = xref.shape[1]
        logpd = torch.empty(n, device=dev)
    traj = torch.empty((n, H, model.L, 13), device=dev) if want_traj else None
    check(_lib.lib().mbd_rollout_traj(model.handle, _p(state_init), _p(Y0s), n, H, _p(rewss), _p(rews), _p(xref), href, _p(logpd),
                                      _p(final), _p(track), nsub_override, _p(traj), _stream()), "mbd_rollout_traj")
    return dict(rews=rews, rewss=rewss, logpd=logpd, final=final, track=track, traj=traj)


def sample_rollout(model: Model, state_init, key, n_total, n_begin, n_local, H, sigma, Ybar, Y0s_out, rews_out,
                   xref=None, logpd_out=None):
    """The fused hot-path kernel: writes Y0s_out [n_local,H*nu], rews_out [n_local] (+logpd_out)."""
    k, kp = key_ptr(key)
    href = 0 if xref is None else xref.shape[1]
    check(_lib.lib().mbd_sample_rollout(model.handle, _p(_dev(state_init)), kp, n_total, n_begin, n_local, H, ctypes.c_float(sigma),
                                        _p(_dev(Ybar)), _p(_dev(Y0s_out)), _p(_dev(rews_out)), _p(xref), href, _p(logpd_out),
                                        _stream()), "mbd_sample_rollout")


def car2d_rollout(params, x0, Y0s, xref=None, want_rewss=False, want_traj=False, key=None, n_total=0, n_begin=0,
                  sigma=0.0, Ybar=None, rews_out=None, logpd_out=None):
    """Car2d rollouts; with `key` the noise is drawn in-kernel and written to Y0s [n,H,2]."""
    params, x0, Y0s = _dev(params), _dev(x0), _dev(Y0s)
    n, H, _ = Y0s.shape
    dev = Y0s.device
    rews = torch.empty(n, device=dev) if rews_out is None else rews_out
    rewss = torch.empty((n, H), device=dev) if want_rewss else None
    traj = torch.empty((n, H, 3), device=dev) if want_traj else None
    logpd, href = None, 0
    if xref is not None:
        href = xref.shape[0]
        logpd = torch.empty(n, device=dev) if logpd_out is None else logpd_out
    kp = None
    if key is not None:
        k, kp = key_ptr(key)
    check(_lib.lib().mbd_car2d_rollout(_p(params), _p(x0), kp, n_total, n_begin, n, H, ctypes.c_float(sigma), _p(Ybar), _p(Y0s),
                                       _p(rewss), _p(rews), _p(xref), href, _p(logpd), _p(traj), _stream()), "mbd_car2d_rollout")
    return dict(rews=rews, rewss=rewss, logpd=logpd, traj=traj)


def pusht_rollout(params, x0, Y0s, want_rewss=False, want_final=False, want_traj=False, key=None, n_total=0, n_begin=0,
                  sigma=0.0, Ybar=None, rews_out=None):
    """pushT rollouts (csrc/pusht.cuh); with `key` the noise is drawn in-kernel and written to Y0s [n,H,2]."""
    params, x0, Y0s = _dev(params), _dev(x0), _dev(Y0s)
    n, H, _ = Y0s.shape
    dev = Y0s.device
    rews = torch.empty(n, device=dev) if rews_out is None else rews_out
    rewss = torch.empty((n, H), device=dev) if want_rewss else None
    final = torch.empty((n, 16), device=dev) if want_final else None
    traj = torch.empty((n, H, 16), device=dev) if want_traj else None
    kp = None
    if key is not None:
        k, kp = key_ptr(key)
    check(_lib.lib().mbd_pusht_rollout(_p(params), _p(x0), kp, n_total, n_begin, n, H, ctypes.c_float(sigma), _p(Ybar), _p(Y0s),
                                       _p(rewss), _p(rews), _p(final), _p(traj), _stream()), "mbd_pusht_rollout")
    return dict(rews=rews, rewss=rewss, final=final, traj=traj, logpd=None)


def softmax_weights(rews_all, logpd_all, n_begin, n_local, temp, rew_xref, weights_out, scalars_out, scratch):
    n_total = rews_all.numel()
    check(_lib.lib().mbd_softmax_weights(_p(_dev(rews_all)), _p(logpd_all), n_total, n_begin, n_local, ctypes.c_float(temp),
                                         ctypes.c_float(rew_xref), _p(_dev(weights_out)), _p(_dev(scalars_out)), _p(_dev(scratch)),
                                         _stream()), "mbd_softmax_weights")


def weighted_sum(weights, Y0s, HNu, scratch, partial_out):
    n_local = weights.numel()
    check(_lib.lib().mbd_weighted_sum(_p(_dev(weights)), _p(_dev(Y0s)), n_local, HNu, _p(_dev(scratch)), _p(_dev(partial_out)),
                                      _stream()), "mbd_weighted_sum")


def weighted_sum_runs(weights, Y0s, HNu, runs_out) -> int:
    """first stage only; returns the number of 64-sample runs written to runs_out [nruns, HNu]"""
    rc = _lib.lib().mbd_weighted_sum_runs(_p(_dev(weights)), _p(_dev(Y0s)), weights.numel(), HNu, _p(_dev(runs_out)), _stream())
    if rc <= 0:
        check(rc if rc < 0 else -1, "mbd_weighted_sum_runs")
    return rc


def weighted_sqerr_sum(weights, Y0s, mu, HNu, scratch, partial_out):
    n_local = weights.numel()
    check(_lib.lib().mbd_weighted_sqerr_sum(_p(_dev(weights)), _p(_dev(Y0s)), _p(_dev(mu)), n_local, HNu, _p(_dev(scratch)),
                                            _p(_dev(partial_out)), _stream()), "mbd_weighted_sqerr_sum")


def update(partials, P, HNu, Ybar_i, coef, out):
    c = (ctypes.c_float * 5)(*[float(v) for v in coef])
    check(_lib.lib().mbd_update(_p(_dev(partials)), P, HNu, _p(_dev(Ybar_i)), c, _p(_dev(out)), _stream()), "mbd_update")


def step_launch(plan: "_lib.StepPlan"):
    """one diffusion step (three launches, parameters in device memory): mbd_step_launch"""
    check(_lib.lib().mbd_step_launch(ctypes.byref(plan), _stream()), "mbd_step_launch")


def batch_step_launch(plan: "_lib.StepPlan", B: int, Ndiffuse: int, temps: Optional[torch.Tensor] = None):
    """one diffusion step of B independent problems in lockstep (mbd_batch_step_launch): every per-problem buffer of `plan`
    holds B consecutive single-problem blocks; temps [B] on the device, or None for plan.temp everywhere"""
    check(_lib.lib().mbd_batch_step_launch(ctypes.byref(plan), int(B), int(Ndiffuse), _p(temps), _stream()), "mbd_batch_step_launch")


def pi_batch_step_launch(plan: "_lib.StepPlan", B: int, Nrefine: int, method: int, temps: Optional[torch.Tensor],
                         bufs: "_lib.PiBufs", tail_only: bool = False):
    """one path-integral refinement step (MPPI / CMA-ES / CEM, `method` = _lib.PI_METHODS[name]) of B problems in lockstep
    (mbd_pi_batch_step_launch), laid out as batch_step_launch; tail_only: launches 2 and 3 on the inputs already in the buffers"""
    check(_lib.lib().mbd_pi_batch_step_launch(ctypes.byref(plan), int(B), int(Nrefine), int(method), _p(temps), ctypes.byref(bufs),
                                              int(bool(tail_only)), _stream()), "mbd_pi_batch_step_launch")


def bbo_batch_step_launch(plan: "_lib.StepPlan", B: int, Ndiffuse: int, fn: int, temps: Optional[torch.Tensor],
                          bufs: "_lib.BboBufs"):
    """one black-box optimisation step (`fn` = _lib.BBO_FNS[name]) of B problems in lockstep (mbd_bbo_batch_step_launch), laid
    out as batch_step_launch with H = 1 and nu = dim"""
    check(_lib.lib().mbd_bbo_batch_step_launch(ctypes.byref(plan), int(B), int(Ndiffuse), int(fn), _p(temps), ctypes.byref(bufs),
                                               _stream()), "mbd_bbo_batch_step_launch")


def mnist_step_launch(plan: "_lib.StepPlan", Ndiffuse: int, bufs: "_lib.MnistBufs"):
    """one MNIST diffusion step (mbd_mnist_step_launch): six launches, parameters read from device tables"""
    check(_lib.lib().mbd_mnist_step_launch(ctypes.byref(plan), int(Ndiffuse), ctypes.byref(bufs), _stream()), "mbd_mnist_step_launch")


def mnist_forward(Y0s: torch.Tensor, bufs: "_lib.MnistBufs", rows: torch.Tensor, Js_out: torch.Tensor, z1_out: Optional[torch.Tensor] = None):
    """Js [n] of the parameter rows Y0s [n, 26506] on the training images `rows` [n_img] (int32); z1_out [n, n_img, 32] optional"""
    _dev(Y0s), _dev(rows, torch.int32), _dev(Js_out)
    if z1_out is not None:
        _dev(z1_out)
    check(_lib.lib().mbd_mnist_forward(_p(Y0s), int(Y0s.shape[0]), ctypes.byref(bufs), _p(rows), int(rows.numel()), _p(Js_out),
                                       _p(z1_out), _stream()), "mbd_mnist_forward")


def mnist_batch_indices(sub_keys: np.ndarray, Ndiffuse: int, n_data: int, N: int, idx_out: torch.Tensor):
    """the minibatch table [Ndiffuse, N] of a solve from the permutation round keys sub_keys [Ndiffuse, 2, 2] (uint32)"""
    _dev(idx_out, torch.int32)
    k = np.ascontiguousarray(sub_keys, dtype=np.uint32)
    L = _lib.lib()
    nbytes = ctypes.c_size_t(0)
    check(L.mbd_mnist_batch_indices(k.ctypes.data_as(_lib.c_u32p), int(Ndiffuse), int(n_data), int(N), None, None,
                                    ctypes.byref(nbytes), _stream()), "mbd_mnist_batch_indices")
    scratch = torch.empty(int(nbytes.value), device=idx_out.device, dtype=torch.uint8)
    check(L.mbd_mnist_batch_indices(k.ctypes.data_as(_lib.c_u32p), int(Ndiffuse), int(n_data), int(N), _p(idx_out), _p(scratch),
                                    ctypes.byref(nbytes), _stream()), "mbd_mnist_batch_indices")
    torch.cuda.current_stream().synchronize()   # the scratch is freed on return


def vec_reset(plan: "_lib.VecPlan", keys: torch.Tensor, dr: "Optional[_lib.VecDr]" = None):
    """env.reset(keys[b]) of every env of a vector-env plan (mbd_vec_reset); keys [B, 2] int32 / uint32 bits on the device.  With
    domain randomisation `dr`: mbd_vec_reset_dr (also episode 0's factors)."""
    k = _p(_dev(keys, torch.int32))
    if dr is None:
        check(_lib.lib().mbd_vec_reset(ctypes.byref(plan), k, _stream()), "mbd_vec_reset")
    else:
        check(_lib.lib().mbd_vec_reset_dr(ctypes.byref(plan), ctypes.byref(dr), k, _stream()), "mbd_vec_reset_dr")


def vec_step(plan: "_lib.VecPlan", dr: "Optional[_lib.VecDr]" = None):
    """one env step of every env with the actions in the plan's buffer (mbd_vec_step: two launches, graph-capturable).  With domain
    randomisation `dr`: mbd_vec_step_dr (also each auto-reset's new factors)."""
    if dr is None:
        check(_lib.lib().mbd_vec_step(ctypes.byref(plan), _stream()), "mbd_vec_step")
    else:
        check(_lib.lib().mbd_vec_step_dr(ctypes.byref(plan), ctypes.byref(dr), _stream()), "mbd_vec_step_dr")


def vec_set_state(plan: "_lib.VecPlan"):
    """observations of the states written into the plan's state buffer; they become the envs' first states (mbd_vec_set_state)"""
    check(_lib.lib().mbd_vec_set_state(ctypes.byref(plan), _stream()), "mbd_vec_set_state")


def vec_world_poses(plan: "_lib.VecPlan", pos: torch.Tensor, rot: torch.Tensor):
    """x.pos [B, L, 3] and x.rot [B, L, 4] of the current states of an xpbd vector env (mbd_vec_world_poses)"""
    check(_lib.lib().mbd_vec_world_poses(ctypes.byref(plan), _p(_dev(pos)), _p(_dev(rot)), _stream()), "mbd_vec_world_poses")


def ppo_act(plan: "_lib.PpoPlan", mode: int):
    """one PPO acting launch (mbd_ppo_act) in mode _lib.PPO_*: the policy of every env, its records or the evaluation return"""
    check(_lib.lib().mbd_ppo_act(ctypes.byref(plan), int(mode), _stream()), "mbd_ppo_act")


def ppo_obs_stats(plan: "_lib.PpoPlan"):
    """running_statistics.update with the rollout's acting observations (mbd_ppo_obs_stats: two launches)"""
    check(_lib.lib().mbd_ppo_obs_stats(ctypes.byref(plan), _stream()), "mbd_ppo_obs_stats")


def ppo_gae(plan: "_lib.PpoPlan"):
    """GAE, the advantage normalisation and the entropy noise of one minibatch (mbd_ppo_gae: one launch)"""
    check(_lib.lib().mbd_ppo_gae(ctypes.byref(plan), _stream()), "mbd_ppo_gae")


def sac_act(plan: "_lib.SacPlan", mode: int):
    """one SAC acting launch (mbd_sac_act) in mode _lib.SAC_*: the policy of every env and its half of the replay rows, or the
    evaluation return"""
    check(_lib.lib().mbd_sac_act(ctypes.byref(plan), int(mode), _stream()), "mbd_sac_act")


def sac_record(plan: "_lib.SacPlan"):
    """the env step's reward, discount, next obs and truncation into the replay rows, and the ring's advance (mbd_sac_record)"""
    check(_lib.lib().mbd_sac_record(ctypes.byref(plan), _stream()), "mbd_sac_record")


def sac_sample(plan: "_lib.SacPlan"):
    """one training step's replay sample: indices, gathered rows and the three noise tensors of every update (mbd_sac_sample)"""
    check(_lib.lib().mbd_sac_sample(ctypes.byref(plan), _stream()), "mbd_sac_sample")


def sac_learn_scratch(O: int, nu: int, batch: int) -> int:
    """floats of the fused SAC update's scratch buffer (mbd_sac_learn_scratch)"""
    return int(_lib.lib().mbd_sac_learn_scratch(int(O), int(nu), int(batch)))


def sac_update(plan: "_lib.SacLearnPlan"):
    """one fused SAC gradient update (mbd_sac_update: two launches): the three losses, Adam on the policy, Q and log alpha, the
    Polyak step, then the update counter advances"""
    check(_lib.lib().mbd_sac_update(ctypes.byref(plan), _stream()), "mbd_sac_update")


def mpc_advance(plan: "_lib.MpcPlan", mode: int):
    """one launch of the receding-horizon controller (mbd_mpc_advance) in mode _lib.MPC_*: ACT executes every problem's plan and
    re-arms its next control step, RECORD logs the env step's reward and state"""
    check(_lib.lib().mbd_mpc_advance(ctypes.byref(plan), int(mode), _stream()), "mbd_mpc_advance")


def mpc_pi_advance(plan: "_lib.MpcPiPlan", mode: int):
    """mpc_advance for a controller that plans with a path-integral baseline (mbd_mpc_pi_advance): ACT also logs the sigma the
    control step ended with and resets the next control step's sigma rows to plan.sigma_warm"""
    check(_lib.lib().mbd_mpc_pi_advance(ctypes.byref(plan), int(mode), _stream()), "mbd_mpc_pi_advance")


def ens_draw(plan: "_lib.EnsDrawPlan"):
    """the planner ensemble of every problem's current control step, drawn on the device (mbd_ens_draw, DESIGN.md §5m)"""
    check(_lib.lib().mbd_ens_draw(ctypes.byref(plan), _stream()), "mbd_ens_draw")


def ens_score(ens_rews: torch.Tensor, worst: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """the score launch of an ensemble step alone (mbd_ens_score): ens_rews [..., K] member returns -> [...] sample returns, the
    ordered mean (worst = 0) or the worst-m score (m = worst); the entry point the score tests drive with constructed returns"""
    ens_rews = _dev(ens_rews)
    K = ens_rews.shape[-1]
    out = torch.empty(ens_rews.shape[:-1], device=ens_rews.device, dtype=torch.float32) if out is None else _dev(out)
    check(_lib.lib().mbd_ens_score(_p(ens_rews), _p(out), int(out.numel()), int(K), int(worst), _stream()), "mbd_ens_score")
    return out


def step_tail_launch(plan: "_lib.StepPlan"):
    """launches 2 and 3 of a step only (statistics + softmax, weighted mean + update) on the inputs already in the plan's
    buffers: mbd_step_tail_launch, the entry point the tail tests drive with constructed returns and samples"""
    check(_lib.lib().mbd_step_tail_launch(ctypes.byref(plan), _stream()), "mbd_step_tail_launch")


def ffma_peak(device: Optional[torch.device] = None, iters: int = 4096) -> float:
    """measured fp32 FFMA throughput of the device in TFLOP/s (the fp32 roofline denominator)"""
    _lib.require_gpu()
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    with torch.cuda.device(dev):
        scratch = torch.empty(1 << 20, device=dev)
        out = ctypes.c_float(0.0)
        check(_lib.lib().mbd_ffma_peak(_p(scratch), int(iters), ctypes.byref(out), _stream()), "mbd_ffma_peak")
    return float(out.value)


class Event:
    """raw CUDA event owned by the library (mbd_event_*): recordable from inside the C launch sequence"""

    def __init__(self):
        self.h = _lib.lib().mbd_event_create()
        if not self.h:
            raise MbdError("mbd_event_create failed")

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            try:
                _lib.lib().mbd_event_destroy(ctypes.c_void_p(h))
            except Exception:  # noqa: BLE001
                pass

    def record(self):
        check(_lib.lib().mbd_event_record(ctypes.c_void_p(self.h), _stream()), "mbd_event_record")

    def synchronize(self):
        check(_lib.lib().mbd_event_sync(ctypes.c_void_p(self.h)), "mbd_event_sync")

    def elapsed_ms(self, later: "Event") -> float:
        return float(_lib.lib().mbd_event_elapsed_ms(ctypes.c_void_p(self.h), ctypes.c_void_p(later.h)))


def step_launch_timed(plan: "_lib.StepPlan", before: Event, mid: Event, mid2: Event, after: Event):
    """events: before the rollout kernel | after it | after the statistics kernel | after the update kernel"""
    check(_lib.lib().mbd_step_launch_ev(ctypes.byref(plan), ctypes.c_void_p(before.h), ctypes.c_void_p(mid.h), ctypes.c_void_p(mid2.h),
                                         ctypes.c_void_p(after.h), _stream()), "mbd_step_launch_ev")
