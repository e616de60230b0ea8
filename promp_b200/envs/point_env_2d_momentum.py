"""MetaPointEnvMomentum (ref: meta_policy_search/envs/point_envs/point_env_2d_momentum.py:7-88): the clipped action is an
acceleration, obs = (position, velocity), sparse reward = max(radius - goal distance, 0).
Dynamics/reward run on the GPU (promp_b200/csrc/envs.cuh: PointMomentum)."""
import numpy as np

from promp_b200 import _lib
from promp_b200.envs.base import MetaEnv, Box

_REWARD = dict(sparse=_lib.REWARD_SPARSE, dense=_lib.REWARD_DENSE, dense_squared=_lib.REWARD_DENSE_SQUARED)


class MetaPointEnvMomentum(MetaEnv):
    env_kind = _lib.ENV_POINT_MOMENTUM
    obs_dim = 4
    act_dim = 2

    def __init__(self, reward_type='sparse', sparse_reward_radius=2):
        assert reward_type in ['dense', 'dense_squared', 'sparse']
        self.reward_type_name = reward_type
        self.reward_type = _REWARD[reward_type]
        self.sparse_reward_radius = sparse_reward_radius
        self.corners = [np.array([-2, -2]), np.array([2, -2]), np.array([-2, 2]), np.array([2, 2])]
        self.observation_space = Box(low=-np.inf, high=np.inf, shape=(4,))
        self.action_space = Box(low=-0.1, high=0.1, shape=(2,))
        self.goal = self.corners[0]

    def sample_tasks(self, n_tasks):
        return [self.corners[idx] for idx in np.random.choice(range(len(self.corners)), size=n_tasks)]     # (:79-80)

    def set_task(self, task):
        self.goal = task

    def get_task(self):
        return self.goal

    def task_vector(self, task):
        return np.asarray(task, dtype=np.float32).reshape(2)

    def host_reset_states(self, n):
        """reset (:44-54): per env uniform(-0.2, 0.2, 2) for the position, then uniform(-0.1, 0.1, 2) for the velocity."""
        out = np.empty((n, 4))
        for i in range(n):
            out[i, :2] = np.random.uniform(-0.2, 0.2, size=(2,))
            out[i, 2:] = np.random.uniform(-0.1, 0.1, size=(2,))
        return out

    def log_diagnostics(self, *args, **kwargs):
        pass

    def __str__(self):
        return 'MetaPointEnvMomentum'
