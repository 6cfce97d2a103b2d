"""Reinforcement-learning baselines of the reference (mbd/rl/train_brax.py) on the device vector env (mbd_b200.envs.vec)."""
