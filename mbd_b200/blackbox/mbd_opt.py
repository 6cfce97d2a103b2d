"""Model-based diffusion as a black-box optimiser — counterpart of upstream mbd/blackbox/mbd_opt.py, same constants and output.

    python -m mbd_b200.blackbox.mbd_opt --fn_name Ackley

Each step of mbd_opt.py's `reverse_once` (lines 64-80) is three launches (`mbd_bbo_batch_step_launch`): (1) k_bbo draws
Y0s = clip(normal(Y0s_rng, (Nsample, dim)) * sigmas[t] + mu_0t, -1, 1) and scores every sample, J = -f(Y0s), folding Js.max()
into a device history; (2) and (3) are the MPPI tail of the path-integral baselines: mean / population std / temperature /
softmax, then mu_0tm1 = sum_n w_n Y0s_n.  All Nexp seeds run as ONE batched solve captured in a CUDA graph; problem b draws the
noise of a stand-alone solve with its own key and reduces in the same order, so it reproduces the B = 1 solve bit for bit.

Ported literally:
  - the schedule (betas = linspace(beta0, betaT, Ndiffuse), sigmas = sqrt(1 - alphas_bar)) is engine.make_schedule;
  - the key chain is `rng = PRNGKey(seed)`, then `rng, Y0s_rng = split(rng)` per step (engine.key_chain(PRNGKey(seed), Ndiffuse));
    the warm-up call at t = 0 discards its carry, so it does not advance the chain;
  - the first step's mean is per sample, mu_0t = normal(PRNGKey(seed), (Nsample, dim)), drawn with the key the first split
    consumes; after that step mu_0t is one row;
  - xs[k] = (k + 1) * Nsample and ys[k] = Js.max() of step t = Ndiffuse - 1 - k; main() saves [xs, mean over seeds of ys].
Declared deviations:
  - the shared statistics kernel keeps MBD's guard std < 1e-4 -> 1; mbd_opt.py:76 has none, so there a zero std gives NaN;
  - cos / sin / exp / sqrt are include/mbd_fp32.h's functions and every sum has the fixed order of csrc/blackbox.cuh, so the
    objective values are not XLA's bits; they are held to a float64 bound instead (tests/bbo_ref.py).  The noise is JAX's bits.
One GPU (the reference is single-device).
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

import mbd_b200
from mbd_b200 import _lib, ops, prng
from mbd_b200.planners.engine import LaunchInputs, StepEngine, key_chain, make_schedule, pack_step_params


@dataclass
class Args:
    fn_name: str = "Rastrigin"  # Ackley, Rastrigin, Levy
    dim: int = 800
    Nexp: int = 6  # seeds 0 .. Nexp - 1
    Nsample: int = 64
    Ndiffuse: int = 100
    temp_sample: float = 1.0
    beta0: float = 1e-4
    betaT: float = 1e-2


# mbd_opt.py:16-20: Ackley is searched on [-5, 10], the others on [-5, 5]
DOMAINS = {"Ackley": (-5.0, 10.0), "Rastrigin": (-5.0, 5.0), "Levy": (-5.0, 5.0)}


def problem_keys(seed: int, Ndiffuse: int):
    """(key chain [Ndiffuse, 2], first-step mean key [2]) of one seed: row t = Y0s_rng of step t, from `rng = PRNGKey(seed)` and
    one split per step; the first step's per-sample mean is drawn with PRNGKey(seed) itself (mbd_opt.py:83-84)"""
    k0 = prng.PRNGKey(seed)
    return key_chain(k0, Ndiffuse), k0


def sample_counts(args: Args) -> np.ndarray:
    """xs of mbd_opt.py:89: the samples drawn after each step, Nsample, 2 Nsample, ..., (Ndiffuse - 1) Nsample"""
    return np.arange(1, args.Ndiffuse, dtype=np.int64) * args.Nsample


class BboEngine(StepEngine):
    """B independent black-box solves of one objective and shape (Nsample, dim, Ndiffuse) stepped in lockstep by ONE
    three-launch step (`mbd_bbo_batch_step_launch`); the solve-level surface of StepEngine (set_step, step, capture,
    check_exchange, solve).  Ybars[b] holds problem b's means (row t = mu_0t of step t, row t - 1 its result; row Ndiffuse - 1 is not
    read: the first step draws its mean per sample from init_keys[b]); rews[b] = J of the last step; best_hist[b][t] = Js.max()
    of step t (-inf before it runs)."""

    def __init__(self, fn_name: str, dim: int, Nsample: int, temps, Ndiffuse: int, device: Optional[torch.device] = None):
        if fn_name not in _lib.BBO_FNS:
            raise KeyError(fn_name)
        if len(temps) < 1:
            raise ValueError("a black-box batch needs at least one problem")
        self.fn_name, self.fn = fn_name, _lib.BBO_FNS[fn_name]
        # no env: launch (1) is the objective, the plan carries no model or table
        super().__init__(LaunchInputs.none(), Nsample, 1, dim, Ndiffuse, False, B=len(temps), temps=temps, device=device)
        self.init_keys = torch.zeros((self.B, 2), device=self.device, dtype=torch.int32)
        self.best_hist = torch.full((self.B, self.Nd), float("-inf"), device=self.device)
        self.x_min, self.x_max = DOMAINS[fn_name]
        self._bufs = _lib.BboBufs(self.init_keys.data_ptr(), self.best_hist.data_ptr(), self.x_min, self.x_max)

    def load_schedule(self, keys, sigmas, init_keys):
        """uploads every problem's key chain keys[b] [Ndiffuse, 2], the shared sigmas [Ndiffuse] and the first-step mean keys
        init_keys[b] [2]; clears best_hist"""
        if not (len(keys) == len(init_keys) == self.B):
            raise ops.MbdError(f"need {self.B} key chains and first-step keys, one per problem")
        if len(sigmas) != self.Nd:
            raise ops.MbdError(f"schedule of {len(sigmas)} steps does not match the engine (Ndiffuse={self.Nd})")
        tab = np.stack([pack_step_params(np.asarray(k, np.uint32), sigmas, None, None) for k in keys])
        self.params.copy_(torch.from_numpy(tab))
        self.init_keys.copy_(torch.from_numpy(np.stack([np.asarray(k, np.uint32) for k in init_keys]).view(np.int32)))
        self.best_hist.fill_(float("-inf"))

    def _launch(self):
        ops.bbo_batch_step_launch(self._plan_c, self.B, self.Nd, self.fn, self.temps, self._bufs)


def check_batch_args(args: Args, seeds: Sequence[int]) -> None:
    """run_exp_batch's argument checks, before anything touches the device"""
    if args.fn_name not in DOMAINS:
        raise KeyError(args.fn_name)
    if len(seeds) < 1:
        raise ValueError("run_exp_batch needs at least one seed")
    if args.Ndiffuse < 2:
        raise ValueError(f"Ndiffuse must be at least 2 (got {args.Ndiffuse}); the reference would run no step")
    import torch.distributed as dist
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 or (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        raise ValueError("run_exp_batch runs on one GPU; it cannot run under WORLD_SIZE > 1")


def run_exp_batch(args: Args, seeds: Sequence[int], log_every: int = 10, progress: bool = False):
    """run_exp of mbd_opt.py for every seed at once, as ONE batched solve captured in a CUDA graph and replayed.
    Returns (xs [Ndiffuse - 1], ys [B, Ndiffuse - 1] = Js.max() per step, mus [B, dim] = the final mean), numpy."""
    check_batch_args(args, seeds)
    eng = BboEngine(args.fn_name, args.dim, args.Nsample, [args.temp_sample] * len(seeds), args.Ndiffuse)
    sigmas = make_schedule(args.beta0, args.betaT, args.Ndiffuse)[3]
    pk = [problem_keys(s, args.Ndiffuse) for s in seeds]
    eng.load_schedule([k for k, _ in pk], sigmas, [k0 for _, k0 in pk])

    def log(t):
        return {"rew": f"{eng.best_hist[:, t].mean().item():.2e}"}   # Js.max(), mean over the seeds
    # the warm-up step of the capture is re-run from the same state: every output is rewritten, best_hist is a max
    eng.solve(log if progress else None, log_every, f"Diffusing x{eng.B}" if progress else None)
    ys = eng.best_hist[:, 1:].flip(1).cpu().numpy()
    mus = eng.Ybars[:, 0].cpu().numpy()
    return sample_counts(args), ys, mus


def run_exp(args: Args, seed: int = 0):
    """mbd_opt.py:run_exp: (xs, ys) of one seed (a batch of one)"""
    xs, ys, _ = run_exp_batch(args, [seed])
    return xs, ys[0]


def result_path(args: Args) -> str:
    """where mbd_opt.py:98-101 saves the curve"""
    return os.path.join(mbd_b200.__path__[0], "..", "results", "bbo", f"{args.fn_name}-{args.dim}d_MBD.npy")


def write_result(xs, ys_mean, path: str) -> np.ndarray:
    """saves [xs, ys] as float32 (2, Ndiffuse - 1), the array mbd_opt.py:99-101 saves"""
    out = np.array([np.asarray(xs, np.float32), np.asarray(ys_mean, np.float32)], dtype=np.float32)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.save(path, out)
    return out


def main(argv=None):
    import tyro
    args = tyro.cli(Args, args=argv)
    xs, ys, _ = run_exp_batch(args, list(range(args.Nexp)), progress=True)
    path = result_path(args)
    write_result(xs, ys.mean(axis=0), path)
    print(f"{args.fn_name}-{args.dim}d: Js.max() {ys.mean(axis=0)[0]:.4e} -> {ys.mean(axis=0)[-1]:.4e} (mean over {args.Nexp} seeds); "
          f"saved {os.path.normpath(path)}")
    return path


if __name__ == "__main__":
    main()
