"""Walker2DRandVelEnv / Walker2DRandDirecEnv - MuJoCo-free analytic surrogates.

Follow the reference (meta_policy_search/envs/mujoco_envs/walker2d_rand_vel.py:6-55, walker2d_rand_direc.py:6-55) for the
interface: obs 17 = qpos[1:] ++ clip(qvel, -10, 10), action 6 in [-1, 1], frame_skip 8 at timestep 0.002 (dt = 0.016),
reset qpos = init_qpos + U(-.005,.005)^9 with init height 1.25, qvel = U(-.005,.005)^9, env_infos {}, and
  RandVel:   goal velocity ~ U(0, 10),  reward = -|forward_vel - goal| + 15 - 1e-3*|a|^2
  RandDirec: direction ~ {-1, +1},      reward = direction * forward_vel + 1 - 1e-3*|a|^2
  done = not (0.8 < height < 2.0 and -1 < angle < 1).
The dynamics are this repo's analytic model (DESIGN.md §3.4; CUDA: promp_b200/csrc/envs.cuh walker::).  Its torso is an
inverted pendulum, so paths end early when the walker falls; MetaSampler(reset_mode='device') samples them in the fused
early-termination kernel, reset_mode='numpy' runs the reference's step loop.
"""
import numpy as np

from promp_b200 import _lib
from promp_b200.envs.base import MetaEnv, Box


class Walker2DRandVelEnv(MetaEnv):
    env_kind = _lib.ENV_WALKER
    reward_type = 1                      # the device kernels read the mode from the task vector (task_vector below)
    mode = 1                             # task vector [goal velocity, 1]
    info_keys = ()
    obs_dim = 17
    act_dim = 6

    def __init__(self, goal_velocity=None):
        self.observation_space = Box(low=-np.inf, high=np.inf, shape=(17,))
        self.action_space = Box(low=-1.0, high=1.0, shape=(6,))
        # the reference draws a task at construction (:8)
        self.set_task(goal_velocity if goal_velocity is not None else self.sample_tasks(1)[0])

    def sample_tasks(self, n_tasks):
        return np.random.uniform(0.0, 10.0, (n_tasks,))        # (:12-13)

    def set_task(self, task):
        self.goal_velocity = task

    def get_task(self):
        return self.goal_velocity

    def task_vector(self, task):
        return np.asarray([task, self.mode], dtype=np.float32)

    def host_reset_states(self, n):
        """reset_model: qpos = init_qpos + U(-.005,.005)^9, qvel = init_qvel + U(-.005,.005)^9.  Like the cheetah's
        (HalfCheetahRandDirecEnv.host_reset_states): the reference draws from each env's own gym `np_random` stream, so
        the n envs are drawn vectorised from the global RNG, every qpos first, then every qvel."""
        out = np.empty((n, 18))
        out[:, :9] = np.random.uniform(low=-.005, high=.005, size=(n, 9))
        out[:, 1] += 1.25                                        # walker2d.xml: rootz ref 1.25
        out[:, 9:] = np.random.uniform(low=-.005, high=.005, size=(n, 9))
        return out

    def log_diagnostics(self, paths, prefix=''):
        """The reference's walker logs nothing of its own (MetaEnv.log_diagnostics, envs/base.py:41-47)."""
        pass

    def __str__(self):
        return 'Walker2DRandVelEnv'


class Walker2DRandDirecEnv(Walker2DRandVelEnv):
    reward_type = 0
    mode = 0                             # task vector [direction, 0]

    def __init__(self, goal_direction=None):
        Walker2DRandVelEnv.__init__(self, goal_direction)

    def sample_tasks(self, n_tasks):
        return np.random.choice((-1.0, 1.0), (n_tasks,))       # walker2d_rand_direc.py:12-13

    def set_task(self, task):
        self.goal_direction = task

    def get_task(self):
        return self.goal_direction

    def __str__(self):
        return 'Walker2DRandDirecEnv'
