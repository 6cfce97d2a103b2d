"""Host restatement of the vector env's episode counters and auto-reset (Brax's AutoResetWrapper(EpisodeWrapper(env)) with
action_repeat = 1, as mbd_vec_step applies them), used by tests/test_vecenv_cpu.py and tests/test_vecenv_gpu.py."""
from __future__ import annotations

import numpy as np


def wrapper_step(done_prev, steps_prev, env_done, episode_length: int):
    """one step of the wrappers on arrays [B]: returns (done, truncation, steps, reset_mask)"""
    done_prev, steps_prev, env_done = (np.asarray(a, np.float32) for a in (done_prev, steps_prev, env_done))
    if episode_length <= 0:
        return env_done, np.zeros_like(env_done), steps_prev + np.float32(1), np.zeros(env_done.shape, bool)
    steps = np.where(done_prev != 0, np.float32(0), steps_prev) + np.float32(1)    # AutoResetWrapper: zeroed where done was set
    reached = steps >= episode_length                                                  # EpisodeWrapper
    done = np.where(reached, np.float32(1), env_done).astype(np.float32)
    trunc = np.where(reached, np.float32(1) - env_done, np.float32(0)).astype(np.float32)
    return done, trunc, steps.astype(np.float32), done != 0
