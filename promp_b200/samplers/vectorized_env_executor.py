"""MetaDeviceEnvExecutor: the vec-env interface of the reference
(meta_policy_search/samplers/vectorized_env_executor.py:7-85: step / reset / set_tasks / num_envs)
with all M*E env states resident on the GPU and stepped by one kernel launch (promp_env_step).
It replaces both MetaIterativeEnvExecutor and MetaParallelEnvExecutor (no worker processes, no pipes).
Used for policies that are not device-resident and for early-terminating envs; the fused
fixed-horizon path (promp_rollout) bypasses it entirely.
"""
import numpy as np

from promp_b200 import _lib


class MetaDeviceEnvExecutor(object):
    def __init__(self, env, meta_batch_size, envs_per_task, max_path_length, device=None):
        import torch
        _lib.require_cuda()
        if not hasattr(env, 'device_spec'):
            raise TypeError("promp_b200 needs a device env (promp_b200.envs.*, wrapped by promp_b200.envs.normalize); "
                            "arbitrary Python envs are not stepped on the CPU (no CPU fallback). Got %r" % (env,))
        self.env = env
        self.spec = env.device_spec()
        self.meta_batch_size, self.envs_per_task = meta_batch_size, envs_per_task
        self.n_envs = meta_batch_size * envs_per_task
        self.max_path_length = max_path_length
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        sd, td = self.spec['state_dim'], self.spec['task_dim']
        f32 = dict(dtype=torch.float32, device=self.device)
        self.state = torch.zeros(self.n_envs, sd, **f32)
        self.ts = torch.zeros(self.n_envs, dtype=torch.int32, device=self.device)
        self.task_params = torch.zeros(self.n_envs, td, **f32)        # expanded per env
        self.task_params_per_task = torch.zeros(meta_batch_size, td, **f32)
        self.tasks = None
        self._obs = torch.zeros(self.n_envs, self.spec['obs_dim'], **f32)
        self._rew = torch.zeros(self.n_envs, **f32)
        self._done = torch.zeros(self.n_envs, dtype=torch.uint8, device=self.device)
        inner_env = getattr(env, '_wrapped_env', env)
        self.info_keys = tuple(getattr(inner_env, 'info_keys', ())) if self.spec['ninfo'] else ()
        self._module = self.spec.get('module')      # a user env (envs/cuda_env.py): its env-step / env-observe kernels
        self._info = torch.zeros(max(len(self.info_keys), 2), self.n_envs, **f32)
        self._dummy_reset = torch.zeros(self.n_envs, sd, **f32)

    @property
    def num_envs(self):
        return self.n_envs

    def set_tasks(self, tasks):
        """vectorized_env_executor.py:54-64.  One launch carries the task vectors (promp_set_tasks): the host does not wait for
        the work already queued, such as the previous iteration's graph replay."""
        assert len(tasks) == self.meta_batch_size
        self.tasks = list(tasks)
        inner = getattr(self.env, '_wrapped_env', self.env)
        vec = np.ascontiguousarray(np.stack([inner.task_vector(t) for t in tasks]), dtype=np.float32)
        assert vec.size == self.task_params_per_task.numel(), "task vectors of %d values, expected %d" % (
            vec.size, self.task_params_per_task.numel())
        _lib.call('promp_set_tasks', self.meta_batch_size, self.spec['task_dim'], self.envs_per_task, vec.ctypes.data,
                  _lib.ptr(self.task_params_per_task), _lib.ptr(self.task_params), _lib.stream())
        if len(tasks):
            self.env.set_task(tasks[-1])

    def _observe(self):
        if self._module is not None:
            _lib.call('promp_env_observe_module', self._module.handle(), self.n_envs, _lib.ptr(self.state), _lib.ptr(self._obs),
                      _lib.stream())
        else:
            _lib.call('promp_env_observe', self.spec['env_kind'], self.n_envs, _lib.ptr(self.state), _lib.ptr(self._obs),
                      _lib.stream())

    def reset(self):
        """vectorized_env_executor.py:66-75: reset states drawn on the host numpy RNG in env order."""
        import torch
        inner = getattr(self.env, '_wrapped_env', self.env)
        states = inner.host_reset_states(self.n_envs).astype(np.float32)
        self.state.copy_(torch.from_numpy(states))
        self.ts.zero_()
        self._observe()
        return list(self._obs.cpu().numpy().astype(np.float64))

    def step(self, actions):
        """vectorized_env_executor.py:25-52 -> (obs, rewards, dones, env_infos), lists of length M*E."""
        import torch
        assert len(actions) == self.num_envs
        if getattr(self, '_per_env_tasks_stale', False):
            self.task_params.copy_(self.task_params_per_task.repeat_interleave(self.envs_per_task, dim=0))
            self._per_env_tasks_stale = False
        act = torch.from_numpy(np.asarray(actions, dtype=np.float32).reshape(self.n_envs, -1)).to(self.device)
        s = self.spec
        _lib.call('promp_env_step_module' if self._module is not None else 'promp_env_step',
                  self._module.handle() if self._module is not None else s['env_kind'], s['reward_type'], s['radius'],
                  int(s.get('normalized', False)), self.n_envs, self.max_path_length,
                  _lib.ptr(self.state), _lib.ptr(self.ts), _lib.ptr(act), _lib.ptr(self.task_params),
                  _lib.ptr(self._dummy_reset), _lib.ptr(self._obs), _lib.ptr(self._rew), _lib.ptr(self._done),
                  _lib.ptr(self._info), _lib.stream())
        dones = self._done.cpu().numpy().astype(bool)
        idx = np.flatnonzero(dones)
        if idx.size:   # done envs are reset with fresh host draws, in env order (:47-50)
            inner = getattr(self.env, '_wrapped_env', self.env)
            new = torch.from_numpy(inner.host_reset_states(idx.size).astype(np.float32)).to(self.device)
            self.state[torch.from_numpy(idx).to(self.device)] = new
            self._observe()
        obs = self._obs.cpu().numpy().astype(np.float64)
        rew = self._rew.cpu().numpy().astype(np.float64)
        if self.info_keys:
            info = self._info.cpu().numpy()
            infos = [{k: float(info[i, n]) for i, k in enumerate(self.info_keys)} for n in range(self.n_envs)]
        else:
            infos = [dict() for _ in range(self.n_envs)]
        return list(obs), list(rew), dones, infos
