"""SwimmerRandVelEnv - MuJoCo-free analytic surrogate.

Follows the reference (meta_policy_search/envs/mujoco_envs/swimmer_rand_vel.py:6-57) for the interface: obs 8 =
qpos[2:] ++ qvel, action 2 in [-1, 1], frame_skip 4 at timestep 0.01 (dt = 0.04), reset qpos = U(-.1,.1)^5,
qvel = U(-.1,.1)^5, tasks = goal velocity ~ U(0.1, 0.2), done = False, env_infos {reward_fwd, reward_ctrl} with
  reward_fwd = |forward_vel - goal|,  reward_ctrl = -1e-4*|a|^2,  reward = reward_fwd + reward_ctrl.
reward_fwd keeps the reference's sign as written: it REWARDS deviating from the goal velocity (a quirk of the reference,
kept so that results stay comparable with it).
The dynamics are this repo's analytic model (DESIGN.md §3.4; CUDA: promp_b200/csrc/envs.cuh swimmer::).
"""
import numpy as np

from promp_b200 import _lib
from promp_b200.envs.base import MetaEnv, Box
from promp_b200.utils import logger


class SwimmerRandVelEnv(MetaEnv):
    """reward = |forward_vel - goal| - 1e-4*|a|^2: as in the reference, the forward term rewards deviating from the goal
    velocity rather than tracking it.  The sign is kept as written so that returns stay comparable with the reference."""
    env_kind = _lib.ENV_SWIMMER
    reward_type = 0
    info_keys = ('reward_fwd', 'reward_ctrl')
    obs_dim = 8
    act_dim = 2

    def __init__(self, goal_vel=None):
        self.observation_space = Box(low=-np.inf, high=np.inf, shape=(8,))
        self.action_space = Box(low=-1.0, high=1.0, shape=(2,))
        # the reference draws a task at construction (:8)
        self.set_task(goal_vel if goal_vel is not None else self.sample_tasks(1)[0])

    def sample_tasks(self, n_tasks):
        return np.random.uniform(0.1, 0.2, (n_tasks,))          # (:12-14)

    def set_task(self, task):
        self.goal_vel = task

    def get_task(self):
        return self.goal_vel

    def task_vector(self, task):
        return np.asarray([task], dtype=np.float32)

    def host_reset_states(self, n):
        """reset_model (:41-46): qpos = U(-.1,.1)^5, qvel = U(-.1,.1)^5, drawn vectorised from the global RNG like the
        cheetah's (HalfCheetahRandDirecEnv.host_reset_states): every qpos first, then every qvel."""
        out = np.empty((n, 10))
        out[:, :5] = np.random.uniform(low=-.1, high=.1, size=(n, 5))
        out[:, 5:] = np.random.uniform(low=-.1, high=.1, size=(n, 5))
        return out

    def log_diagnostics(self, paths, prefix=''):
        """(:48-57): progress of observation[-3] (qvel[2], the body's angular velocity, as the reference indexes it)
        between the first and last step of every path."""
        phase = getattr(paths[0], 'phase', None) if len(paths) else None
        if phase is not None and type(phase).__name__ == 'PhaseData':       # fixed-horizon device phase: one reduction
            for k, v in zip(self.DEVICE_LOG_KEYS, self.device_log_terms(phase).cpu().numpy()):
                logger.logkv(prefix + k, float(v))
            return
        progs = [path["observations"][-1][-3] - path["observations"][0][-3] for path in paths]
        logger.logkv(prefix + 'AverageForwardProgress', np.mean(progs))
        logger.logkv(prefix + 'MaxForwardProgress', np.max(progs))
        logger.logkv(prefix + 'MinForwardProgress', np.min(progs))
        logger.logkv(prefix + 'StdForwardProgress', np.std(progs))

    DEVICE_LOG_KEYS = ('AverageForwardProgress', 'MaxForwardProgress', 'MinForwardProgress', 'StdForwardProgress')

    def device_log_terms(self, phase):
        import torch
        obs = phase.obs.view(-1, phase.H, phase.obs_dim)
        progs = (obs[:, -1, -3] - obs[:, 0, -3]).double()
        return torch.stack([progs.mean(), progs.max(), progs.min(), torch.std(progs, unbiased=False)])

    def __str__(self):
        return 'SwimmerRandVelEnv'
