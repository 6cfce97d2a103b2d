"""ctypes binding of libmbd_b200.so (the C ABI in include/mbd_b200.h).

The product path has NO CPU fallback: if the library is missing and cannot be built, or no
CUDA device is present when a device entry point is called, this module raises.

Each ctypes.Structure below mirrors the C struct named by its `_c_name_`, and the integer constants mirror the headers' MBD_*
values; tests/test_abi.py compiles all of them against include/.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import build as _build

_LIB = None
c_f32p = ctypes.POINTER(ctypes.c_float)
c_u32p = ctypes.POINTER(ctypes.c_uint32)
c_i32p = ctypes.POINTER(ctypes.c_int32)
c_vp = ctypes.c_void_p


class MbdError(RuntimeError):
    pass


class StepParams(ctypes.Structure):
    """mbd_step_params (include/mbd_b200.h): one row per diffusion step index, 32 bytes"""
    _c_name_ = "mbd_step_params"
    _fields_ = [("key", ctypes.c_uint32 * 2), ("sigma", ctypes.c_float), ("coef", ctypes.c_float * 5)]


class StepPlan(ctypes.Structure):
    """mbd_step_plan (include/mbd_b200.h), field for field"""
    _c_name_ = "mbd_step_plan"
    _fields_ = [
        ("model", c_vp), ("car_params_dev", c_vp), ("state_init_dev", c_vp), ("params_dev", c_vp), ("ctl_dev", c_vp),
        ("Ybars_dev", c_vp), ("rew_hist_dev", c_vp),
        ("n_total", ctypes.c_int32), ("n_begin", ctypes.c_int32), ("n_local", ctypes.c_int32), ("H", ctypes.c_int32), ("nu", ctypes.c_int32),
        ("temp", ctypes.c_float), ("rew_xref", ctypes.c_float),
        ("xref_dev", c_vp), ("href", ctypes.c_int32), ("env_kind", ctypes.c_int32),
        ("Y0s_dev", c_vp), ("rews_dev", c_vp), ("logpd_dev", c_vp), ("rews_all_dev", c_vp), ("logpd_all_dev", c_vp), ("logp_dev", c_vp),
        ("weights_dev", c_vp), ("runs_dev", c_vp), ("partial_dev", c_vp), ("scalars_dev", c_vp),
        ("P", ctypes.c_int32), ("rank", ctypes.c_int32),
        ("peer_base_ptrs", ctypes.POINTER(ctypes.c_uint64)),
        ("off_rews_words", ctypes.c_uint64), ("off_logpd_words", ctypes.c_uint64), ("off_partial_words", ctypes.c_uint64),
        ("off_flags_words", ctypes.c_uint64), ("timeout_cycles", ctypes.c_uint64),
        ("ens_factors_dev", c_vp), ("ens_rews_dev", c_vp), ("ens_k", ctypes.c_int32), ("ens_worst", ctypes.c_int32),
    ]


class PiBufs(ctypes.Structure):
    """mbd_pi_bufs (include/mbd_b200.h): the buffers the path-integral update rules add to a step plan"""
    _c_name_ = "mbd_pi_bufs"
    _fields_ = [("sigma_hist_dev", c_vp), ("cma_scratch_dev", c_vp), ("cem_idx_dev", c_vp)]


class BboBufs(ctypes.Structure):
    """mbd_bbo_bufs (include/mbd_b200.h): what a black-box step adds to a step plan"""
    _c_name_ = "mbd_bbo_bufs"
    _fields_ = [("init_keys_dev", c_vp), ("best_hist_dev", c_vp), ("x_min", ctypes.c_float), ("x_max", ctypes.c_float)]


class MnistBufs(ctypes.Structure):
    """mbd_mnist_bufs (include/mbd_b200.h): what an MNIST step adds to a step plan"""
    _c_name_ = "mbd_mnist_bufs"
    _fields_ = [("train_images_dev", c_vp), ("train_labels_dev", c_vp), ("test_images_dev", c_vp), ("test_labels_dev", c_vp),
                ("keys_dev", c_vp), ("batch_idx_dev", c_vp), ("acc_hist_dev", c_vp), ("layers", ctypes.c_int32 * 4),
                ("n_train", ctypes.c_int32), ("n_test", ctypes.c_int32), ("eval_every", ctypes.c_int32)]


class VecPlan(ctypes.Structure):
    """mbd_vec_plan (include/mbd_b200.h): a batch of envs stepped together on the device"""
    _c_name_ = "mbd_vec_plan"
    _fields_ = [("kind", ctypes.c_int32), ("B", ctypes.c_int32), ("model", c_vp), ("params_dev", c_vp), ("kin_dev", c_vp),
                ("reset_dev", c_vp), ("obs_layout", ctypes.c_int32), ("done_rule", ctypes.c_int32), ("episode_length", ctypes.c_int32),
                ("nq", ctypes.c_int32), ("nqd", ctypes.c_int32), ("nu", ctypes.c_int32),
                ("state_dev", c_vp), ("next_state_dev", c_vp), ("first_state_dev", c_vp), ("actions_dev", c_vp), ("obs_dev", c_vp),
                ("first_obs_dev", c_vp), ("reward_dev", c_vp), ("done_dev", c_vp), ("truncation_dev", c_vp), ("steps_dev", c_vp),
                ("factors_dev", c_vp)]


class VecDr(ctypes.Structure):
    """mbd_vec_dr (include/mbd_b200.h): domain randomisation of a vector env's factor table"""
    _c_name_ = "mbd_vec_dr"
    _fields_ = [("keys_dev", c_vp), ("episodes_dev", c_vp), ("range", ctypes.c_float * 4)]


class PpoPlan(ctypes.Structure):
    """mbd_ppo_plan (include/mbd_b200.h): the PPO acting step, observation statistics and GAE"""
    _c_name_ = "mbd_ppo_plan"
    _fields_ = [("B", ctypes.c_int32), ("O", ctypes.c_int32), ("nu", ctypes.c_int32), ("slots", ctypes.c_int32),
                ("unroll", ctypes.c_int32), ("mb", ctypes.c_int32), ("reward_scaling", ctypes.c_float), ("discount", ctypes.c_float),
                ("gae_lambda", ctypes.c_float), ("act_key_rows", ctypes.c_int32), ("loss_key_rows", ctypes.c_int32),
                ("policy_dev", c_vp), ("mean_dev", c_vp), ("std_dev", c_vp), ("act_keys_dev", c_vp), ("act_ctl_dev", c_vp),
                ("env_obs_dev", c_vp), ("env_reward_dev", c_vp), ("env_done_dev", c_vp), ("env_trunc_dev", c_vp),
                ("env_actions_dev", c_vp), ("obs_dev", c_vp), ("raw_dev", c_vp), ("logp_dev", c_vp), ("reward_dev", c_vp),
                ("disc_dev", c_vp), ("trunc_dev", c_vp), ("ret_dev", c_vp), ("active_dev", c_vp), ("stat_dev", c_vp),
                ("stat_scratch_dev", c_vp), ("loss_keys_dev", c_vp), ("loss_ctl_dev", c_vp), ("traj_dev", c_vp), ("values_dev", c_vp),
                ("vs_dev", c_vp), ("adv_dev", c_vp), ("ent_eps_dev", c_vp)]


class SacPlan(ctypes.Structure):
    """mbd_sac_plan (include/mbd_b200.h): the SAC acting step, the replay record and the replay sampler"""
    _c_name_ = "mbd_sac_plan"
    _fields_ = [("B", ctypes.c_int32), ("O", ctypes.c_int32), ("nu", ctypes.c_int32), ("capacity", ctypes.c_int32),
                ("batch", ctypes.c_int32), ("updates", ctypes.c_int32), ("act_key_rows", ctypes.c_int32), ("noise_key_rows", ctypes.c_int32),
                ("policy_dev", c_vp), ("mean_dev", c_vp), ("std_dev", c_vp), ("act_keys_dev", c_vp), ("act_ctl_dev", c_vp),
                ("env_obs_dev", c_vp), ("env_reward_dev", c_vp), ("env_done_dev", c_vp), ("env_trunc_dev", c_vp),
                ("env_actions_dev", c_vp), ("ret_dev", c_vp), ("active_dev", c_vp), ("stage_obs_dev", c_vp), ("ring_dev", c_vp),
                ("ring_ctl_dev", c_vp), ("sample_ctl_dev", c_vp), ("noise_keys_dev", c_vp), ("idx_dev", c_vp), ("batch_dev", c_vp),
                ("eps_dev", c_vp)]


class SacLearnPlan(ctypes.Structure):
    """mbd_sac_learn_plan (include/mbd_b200.h): the fused SAC gradient update"""
    _c_name_ = "mbd_sac_learn_plan"
    _fields_ = [("O", ctypes.c_int32), ("nu", ctypes.c_int32), ("batch", ctypes.c_int32), ("updates", ctypes.c_int32),
                ("learning_rate", ctypes.c_float), ("reward_scaling", ctypes.c_float), ("discounting", ctypes.c_float),
                ("tau", ctypes.c_float), ("policy_dev", c_vp), ("q_dev", c_vp), ("target_q_dev", c_vp), ("log_alpha_dev", c_vp),
                ("policy_m_dev", c_vp), ("policy_v_dev", c_vp), ("q_m_dev", c_vp), ("q_v_dev", c_vp), ("alpha_mv_dev", c_vp),
                ("ctl_dev", c_vp), ("mean_dev", c_vp), ("std_dev", c_vp), ("batch_dev", c_vp), ("eps_dev", c_vp),
                ("upd_ctl_dev", c_vp), ("scratch_dev", c_vp), ("scratch_floats", ctypes.c_int64), ("losses_dev", c_vp)]


class MpcPlan(ctypes.Structure):
    """mbd_mpc_plan (include/mbd_b200.h): the step between two control steps of the receding-horizon controller"""
    _c_name_ = "mbd_mpc_plan"
    _fields_ = [("B", ctypes.c_int32), ("H", ctypes.c_int32), ("nu", ctypes.c_int32), ("Ndiffuse", ctypes.c_int32),
                ("Nwarm", ctypes.c_int32), ("Nstep", ctypes.c_int32), ("state_words", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("params_dev", c_vp), ("ctl_dev", c_vp), ("Ybars_dev", c_vp), ("rew_hist_dev", c_vp), ("keys_dev", c_vp),
                ("mpc_ctl_dev", c_vp), ("env_actions_dev", c_vp), ("env_state_dev", c_vp), ("env_reward_dev", c_vp),
                ("actions_dev", c_vp), ("rewards_dev", c_vp), ("states_dev", c_vp), ("rew_hist_log_dev", c_vp)]


class MpcPiPlan(ctypes.Structure):
    """mbd_mpc_pi_plan (include/mbd_b200.h): mbd_mpc_plan for a path-integral baseline, plus the sigma reset and its log"""
    _c_name_ = "mbd_mpc_pi_plan"
    _fields_ = [("base", MpcPlan), ("sigma_warm", ctypes.c_float), ("pad", ctypes.c_int32), ("sigma_log_dev", c_vp)]


class EnsDrawPlan(ctypes.Structure):
    """mbd_ens_draw_plan (include/mbd_b200.h): the planner ensemble drawn afresh at every control step"""
    _c_name_ = "mbd_ens_draw_plan"
    _fields_ = [("B", ctypes.c_int32), ("K", ctypes.c_int32), ("Nstep", ctypes.c_int32), ("pad", ctypes.c_int32),
                ("keys_dev", c_vp), ("ranges_dev", c_vp), ("mpc_ctl_dev", c_vp), ("ens_factors_dev", c_vp)]


MPC_ACT, MPC_RECORD = 0, 1                                     # MBD_MPC_*
PPO_ACT, PPO_RECORD, PPO_EVAL, PPO_EVAL_RECORD = 0, 1, 2, 3   # MBD_PPO_*
PPO_MAX_OBS, PPO_MAX_NU, PPO_MAX_MB, PPO_STAT_ROWS = 128, 32, 4096, 256
SAC_ACT, SAC_EVAL, SAC_EVAL_RECORD = 0, 1, 2                   # MBD_SAC_*
SAC_MAX_CAPACITY, SAC_HIDDEN = 1 << 24, 256
SAC_LEARN_MAX_BATCH = 4096                                     # MBD_SAC_LEARN_MAX_BATCH

VEC_XPBD, VEC_CAR2D, VEC_PUSHT = 0, 1, 2                                   # MBD_VEC_*
VEC_OBS = {"qqd": 0, "hopper": 1, "skip2": 2, "skip1": 3, "state": 4}     # MBD_VEC_OBS_*
VEC_DONE_ZERO, VEC_DONE_COUNTER, VEC_DONE_PUSHT = 0, 1, 2                 # MBD_VEC_DONE_*
VEC_RESET = {"none": 0, "uniform": 1, "normal": 2, "pusht": 3, "const": 4}  # MBD_VEC_RESET_*
VEC_RT_Q = 8             # MBD_VEC_RT_Q: first init_q word of the reset table
VEC_MAX_B = 65536        # MBD_VEC_MAX_B
K64_WORDS = 920          # MBD_K64_WORDS (include/mbd_kin64.h)

MNIST_HNU = 26506        # MBD_MNIST_HNU
BBO_FNS = {"Ackley": 1, "Rastrigin": 2, "Levy": 3}   # MBD_BBO_ACKLEY / MBD_BBO_RASTRIGIN / MBD_BBO_LEVY
PI_METHODS = {"mppi": 1, "cma-es": 2, "cem": 3}   # MBD_PI_MPPI / MBD_PI_CMAES / MBD_PI_CEM
PI_IDX_STRIDE = 16       # MBD_PI_IDX_STRIDE: ints per problem in cem_idx (10 picks, then the count)
PI_TOPK = 10
ENS_MAXK = 16            # MBD_ENS_MAXK: members of a planner ensemble

STEP_PARAMS_WORDS = 8    # sizeof(mbd_step_params) / 4
STEP_CTL_WORDS = 32      # sizeof(mbd_step_ctl) / 4
ENV_CAR2D, ENV_PUSHT = 0, 1   # mbd_step_plan.env_kind (model == NULL)


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.OUT
    # Build when the library is missing OR was built from other sources (content hash stored beside the .so: copied
    # trees carry arbitrary mtimes, so mtimes are not consulted).  build(force=False) re-checks inside an exclusive file
    # lock, so of N ranks starting together exactly one compiles and the others load the finished file.
    if _build.is_stale():
        try:
            path = _build.build(force=False)
        except Exception as e:  # noqa: BLE001
            raise MbdError(f"libmbd_b200.so is missing or stale and could not be built ({e}); there is no CPU fallback") from e
    L = ctypes.CDLL(path)
    L.mbd_last_error.restype = ctypes.c_char_p
    L.mbd_device_count.restype = ctypes.c_int
    L.mbd_model_create.restype = c_vp
    L.mbd_model_create.argtypes = [c_u32p, ctypes.c_size_t]
    L.mbd_model_destroy.argtypes = [c_vp]
    L.mbd_sample.argtypes = [c_u32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, c_vp, c_vp, c_vp]
    L.mbd_rollout.argtypes = [c_vp, c_vp, c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, ctypes.c_int, c_vp, c_vp, c_vp,
                              ctypes.c_int, c_vp]
    L.mbd_rollout_traj.argtypes = [c_vp, c_vp, c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, ctypes.c_int, c_vp, c_vp, c_vp,
                                   ctypes.c_int, c_vp, c_vp]
    L.mbd_sample_rollout.argtypes = [c_vp, c_vp, c_u32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                     c_vp, c_vp, c_vp, c_vp, ctypes.c_int, c_vp, c_vp]
    L.mbd_car2d_rollout.argtypes = [c_vp, c_vp, c_u32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                    c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_int, c_vp, c_vp, c_vp]
    L.mbd_pusht_rollout.argtypes = [c_vp, c_vp, c_u32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                    c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.mbd_softmax_weights.argtypes = [c_vp, c_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                      c_vp, c_vp, c_vp, c_vp]
    L.mbd_weighted_sum.argtypes = [c_vp, c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp]
    L.mbd_weighted_sum_runs.argtypes = [c_vp, c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp]
    L.mbd_weighted_sqerr_sum.argtypes = [c_vp, c_vp, c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp]
    L.mbd_test_arith.argtypes = [ctypes.c_int, c_vp, c_vp, c_vp, ctypes.c_int, c_vp]
    L.mbd_test_err.argtypes = [ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, ctypes.c_int, c_vp]
    L.mbd_test_sweep.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_float,
                                 ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, c_vp]
    L.mbd_update.argtypes = [c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_f32p, c_vp, c_vp]
    L.mbd_step_launch.argtypes = [ctypes.POINTER(StepPlan), c_vp]
    L.mbd_step_tail_launch.argtypes = [ctypes.POINTER(StepPlan), c_vp]
    L.mbd_batch_step_launch.argtypes = [ctypes.POINTER(StepPlan), ctypes.c_int, ctypes.c_int, c_vp, c_vp]
    L.mbd_pi_batch_step_launch.argtypes = [ctypes.POINTER(StepPlan), ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp,
                                           ctypes.POINTER(PiBufs), ctypes.c_int, c_vp]
    L.mbd_ens_score.argtypes = [c_vp, c_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp]
    L.mbd_ens_draw.argtypes = [ctypes.POINTER(EnsDrawPlan), c_vp]
    L.mbd_bbo_batch_step_launch.argtypes = [ctypes.POINTER(StepPlan), ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp,
                                            ctypes.POINTER(BboBufs), c_vp]
    L.mbd_mnist_step_launch.argtypes = [ctypes.POINTER(StepPlan), ctypes.c_int, ctypes.POINTER(MnistBufs), c_vp]
    L.mbd_mnist_forward.argtypes = [c_vp, ctypes.c_int, ctypes.POINTER(MnistBufs), c_vp, ctypes.c_int, c_vp, c_vp, c_vp]
    L.mbd_mnist_batch_indices.argtypes = [c_u32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp, c_vp,
                                          ctypes.POINTER(ctypes.c_size_t), c_vp]
    L.mbd_vec_reset.argtypes = [ctypes.POINTER(VecPlan), c_vp, c_vp]
    L.mbd_vec_step.argtypes = [ctypes.POINTER(VecPlan), c_vp]
    L.mbd_vec_set_state.argtypes = [ctypes.POINTER(VecPlan), c_vp]
    L.mbd_vec_world_poses.argtypes = [ctypes.POINTER(VecPlan), c_vp, c_vp, c_vp]
    L.mbd_vec_reset_dr.argtypes = [ctypes.POINTER(VecPlan), ctypes.POINTER(VecDr), c_vp, c_vp]
    L.mbd_vec_step_dr.argtypes = [ctypes.POINTER(VecPlan), ctypes.POINTER(VecDr), c_vp]
    L.mbd_ppo_act.argtypes = [ctypes.POINTER(PpoPlan), ctypes.c_int, c_vp]
    L.mbd_ppo_obs_stats.argtypes = [ctypes.POINTER(PpoPlan), c_vp]
    L.mbd_ppo_gae.argtypes = [ctypes.POINTER(PpoPlan), c_vp]
    L.mbd_sac_act.argtypes = [ctypes.POINTER(SacPlan), ctypes.c_int, c_vp]
    L.mbd_sac_record.argtypes = [ctypes.POINTER(SacPlan), c_vp]
    L.mbd_sac_sample.argtypes = [ctypes.POINTER(SacPlan), c_vp]
    L.mbd_sac_learn_scratch.restype = ctypes.c_int64
    L.mbd_sac_learn_scratch.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.mbd_sac_update.argtypes = [ctypes.POINTER(SacLearnPlan), c_vp]
    L.mbd_mpc_advance.argtypes = [ctypes.POINTER(MpcPlan), ctypes.c_int, c_vp]
    L.mbd_mpc_pi_advance.argtypes = [ctypes.POINTER(MpcPiPlan), ctypes.c_int, c_vp]
    L.mbd_step_launch_ev.argtypes =[ctypes.POINTER(StepPlan), c_vp, c_vp, c_vp, c_vp, c_vp]
    L.mbd_event_create.restype = c_vp
    L.mbd_event_destroy.argtypes = [c_vp]
    L.mbd_event_record.argtypes = [c_vp, c_vp]
    L.mbd_event_sync.argtypes = [c_vp]
    L.mbd_event_elapsed_ms.restype = ctypes.c_float
    L.mbd_event_elapsed_ms.argtypes = [c_vp, c_vp]
    L.mbd_ffma_peak.argtypes = [c_vp, ctypes.c_int, c_f32p, c_vp]
    _LIB = L
    return L


EXPORTS = ["mbd_set_kernel_variant", "mbd_set_prng_layout", "mbd_model_set_warp_order", "mbd_last_error", "mbd_device_count", "mbd_model_create", "mbd_model_destroy", "mbd_sample",
           "mbd_rollout", "mbd_rollout_traj", "mbd_sample_rollout", "mbd_car2d_rollout", "mbd_pusht_rollout", "mbd_softmax_weights", "mbd_weighted_sum", "mbd_weighted_sum_runs", "mbd_weighted_sqerr_sum", "mbd_test_arith", "mbd_test_err", "mbd_test_sweep","mbd_update", "mbd_step_launch", "mbd_batch_step_launch", "mbd_pi_batch_step_launch", "mbd_ens_score", "mbd_ens_draw", "mbd_bbo_batch_step_launch", "mbd_mnist_step_launch", "mbd_mnist_forward", "mbd_mnist_batch_indices", "mbd_vec_reset", "mbd_vec_step", "mbd_vec_set_state", "mbd_vec_world_poses", "mbd_vec_reset_dr", "mbd_vec_step_dr", "mbd_ppo_act", "mbd_ppo_obs_stats", "mbd_ppo_gae", "mbd_sac_act", "mbd_sac_record", "mbd_sac_sample", "mbd_sac_learn_scratch", "mbd_sac_update", "mbd_mpc_advance", "mbd_mpc_pi_advance", "mbd_step_tail_launch", "mbd_step_launch_ev", "mbd_event_create", "mbd_event_destroy", "mbd_event_record",
           "mbd_event_sync", "mbd_event_elapsed_ms", "mbd_ffma_peak"]


def check(rc: int, what: str):
    if rc != 0:
        raise MbdError(f"{what} failed (rc={rc}): {lib().mbd_last_error().decode()}")


def key_ptr(key):
    k = np.ascontiguousarray(key, dtype=np.uint32)
    return k, k.ctypes.data_as(c_u32p)


def require_gpu():
    if lib().mbd_device_count() <= 0:
        raise MbdError("no CUDA device visible: the MBD hot path has no CPU fallback")
