"""MetaPointEnvCorner (ref: meta_policy_search/envs/point_envs/point_env_2d_corner.py:7-93).
Dynamics/reward run on the GPU (promp_b200/csrc/envs.cuh: PointCorner)."""
import numpy as np

from promp_b200 import _lib
from promp_b200.envs.base import MetaEnv, Box

_REWARD = dict(sparse=_lib.REWARD_SPARSE, dense=_lib.REWARD_DENSE, dense_squared=_lib.REWARD_DENSE_SQUARED)


class MetaPointEnvCorner(MetaEnv):
    env_kind = _lib.ENV_POINT_CORNER
    obs_dim = 2
    act_dim = 2

    def __init__(self, reward_type='sparse', sparse_reward_radius=0.5):
        assert reward_type in ['dense', 'dense_squared', 'sparse']
        self.reward_type_name = reward_type
        self.reward_type = _REWARD[reward_type]
        self.sparse_reward_radius = sparse_reward_radius
        self.corners = [np.array([-2, -2]), np.array([2, -2]), np.array([-2, 2]), np.array([2, 2])]
        self.observation_space = Box(low=-np.inf, high=np.inf, shape=(2,))
        self.action_space = Box(low=-0.2, high=0.2, shape=(2,))
        self.goal = self.corners[0]

    def sample_tasks(self, n_tasks):
        # same single numpy draw as the reference (:86-87)
        return [self.corners[idx] for idx in np.random.choice(range(len(self.corners)), size=n_tasks)]

    def set_task(self, task):
        self.goal = task

    def get_task(self):
        return self.goal

    def task_vector(self, task):
        return np.asarray(task, dtype=np.float32).reshape(2)

    def host_reset_states(self, n):
        # reset (:43-52): one uniform(-0.2, 0.2, size=2) per env, in env order
        return np.random.uniform(-0.2, 0.2, size=(n, 2))

    def log_diagnostics(self, *args, **kwargs):
        pass
