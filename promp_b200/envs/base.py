"""MetaEnv interface (ref: meta_policy_search/envs/base.py:6-49) for device-resident envs.

A device env is a *description*: its dynamics run inside the CUDA kernels (promp_rollout /
promp_env_step), selected by `device_spec()`.  Task sampling stays on the host numpy RNG so that
`np.random.seed(s)` reproduces the reference's task sequence draw for draw.
"""
import numpy as np

from promp_b200 import _lib


class Box(object):
    """Just enough of gym.spaces.Box (gym 0.10.5: float32 bounds by default)."""

    def __init__(self, low, high, shape=None, dtype=np.float32):
        if shape is None:
            low, high = np.asarray(low), np.asarray(high)
            shape = low.shape
        else:
            low = low + np.zeros(shape)
            high = high + np.zeros(shape)
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)
        self.low = np.asarray(low).astype(dtype)
        self.high = np.asarray(high).astype(dtype)


class MetaEnv(object):
    """Subclasses define: env_kind, obs_dim, act_dim, observation_space, action_space,
    sample_tasks / set_task / get_task, task_vector(task) and host_reset_states(n)."""
    env_kind = None
    reward_type = _lib.REWARD_SPARSE
    sparse_reward_radius = 0.5

    def sample_tasks(self, n_tasks):
        raise NotImplementedError

    def set_task(self, task):
        raise NotImplementedError

    def get_task(self):
        raise NotImplementedError

    def log_diagnostics(self, paths, prefix=''):
        pass

    DEVICE_LOG_KEYS = ()

    def device_log_terms(self, phase):
        return None

    # ---- device description -------------------------------------------------------------
    def device_spec(self):
        """env_kind (a built-in) or module (a user env, envs/cuda_env.py); ends_early: paths end on `done`; ninfo: env-info
        channels the kernels write."""
        info = len(getattr(self, 'info_keys', ('reward_run', 'reward_ctrl'))) if self.env_kind in _lib.INFO_ENVS else 0
        return dict(env_kind=self.env_kind, reward_type=self.reward_type, radius=float(self.sparse_reward_radius),
                    obs_dim=self.obs_dim, act_dim=self.act_dim,
                    state_dim=_lib.load().promp_env_state_dim(self.env_kind),
                    task_dim=_lib.load().promp_env_task_dim(self.env_kind),
                    ends_early=self.env_kind in _lib.EARLY_TERM_ENVS, ninfo=info)

    def task_vector(self, task):
        """float32 vector handed to the kernels for one task."""
        raise NotImplementedError

    def host_reset_states(self, n):
        """[n, state_dim] reset states drawn from the global numpy RNG in the reference's order."""
        raise NotImplementedError

    # ---- single-env gym-style API, executed by the same device kernels (batch of one) ----
    def _single(self):
        if getattr(self, '_single_exec', None) is None:
            from promp_b200.samplers.vectorized_env_executor import MetaDeviceEnvExecutor
            self._single_exec = MetaDeviceEnvExecutor(self, 1, 1, max_path_length=2 ** 30)
        return self._single_exec

    def reset(self):
        ex = self._single()
        ex.set_tasks([self.get_task()])
        return ex.reset()[0]

    def step(self, action):
        ex = self._single()
        obs, rewards, dones, infos = ex.step([np.asarray(action)])
        return obs[0], rewards[0], bool(dones[0]), infos[0]
