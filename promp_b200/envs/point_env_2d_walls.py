"""MetaPointEnvWalls (ref: meta_policy_search/envs/point_envs/point_env_2d_walls.py:7-117): two circular walls of radius 1
and 2 around the origin, each passable only within distance 1 of its gap centre; tasks = goal corner + the two gaps.
Dynamics/reward run on the GPU (promp_b200/csrc/envs.cuh: PointWalls)."""
import numpy as np

from promp_b200 import _lib
from promp_b200.envs.base import MetaEnv, Box

_REWARD = dict(dense=_lib.REWARD_DENSE, dense_squared=_lib.REWARD_DENSE_SQUARED)


class MetaPointEnvWalls(MetaEnv):
    env_kind = _lib.ENV_POINT_WALLS
    obs_dim = 2
    act_dim = 2

    def __init__(self, reward_type='dense', sparse_reward_radius=2):
        assert reward_type in ['dense', 'dense_squared', 'sparse']
        if reward_type == 'sparse':
            # the reference's sparse branch returns None outside the radius (:86-89) and cannot be sampled either
            raise NotImplementedError("MetaPointEnvWalls: reward_type 'sparse' returns None in the reference; use dense / dense_squared")
        self.reward_type_name = reward_type
        self.reward_type = _REWARD[reward_type]
        self.sparse_reward_radius = sparse_reward_radius
        self.corners = [np.array([-2, -2]), np.array([2, -2]), np.array([-2, 2]), np.array([2, 2])]
        self.observation_space = Box(low=-np.inf, high=np.inf, shape=(2,))
        self.action_space = Box(low=-0.2, high=0.2, shape=(2,))
        self.goal, self.gap_1, self.gap_2 = self.corners[0], np.array([1.0, 0.0]), np.array([2.0, 0.0])

    def sample_tasks(self, n_tasks):
        # the reference's three numpy draws in the same order (:102-108)
        goals = [self.corners[idx] for idx in np.random.choice(range(len(self.corners)), size=n_tasks)]
        gaps_1 = np.random.normal(size=(n_tasks, 2))
        gaps_1 /= np.linalg.norm(gaps_1, axis=1)[..., np.newaxis]
        gaps_2 = np.random.normal(size=(n_tasks, 2))
        gaps_2 /= (np.linalg.norm(gaps_2, axis=1) / 2)[..., np.newaxis]
        return [dict(goal=goal, gap_1=gap_1, gap_2=gap_2) for goal, gap_1, gap_2 in zip(goals, gaps_1, gaps_2)]

    def set_task(self, task):
        self.goal, self.gap_1, self.gap_2 = task['goal'], task['gap_1'], task['gap_2']

    def get_task(self):
        return dict(goal=self.goal, gap_1=self.gap_1, gap_2=self.gap_2)

    def task_vector(self, task):
        return np.concatenate([np.asarray(task[k], dtype=np.float32).reshape(2) for k in ('goal', 'gap_1', 'gap_2')])

    def host_reset_states(self, n):
        return np.random.uniform(-0.2, 0.2, size=(n, 2))          # reset (:53-62)

    def log_diagnostics(self, *args, **kwargs):
        pass

    def __str__(self):
        return 'MetaPointEnvWalls'
