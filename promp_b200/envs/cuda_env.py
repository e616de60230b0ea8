"""Users' own environments on the device: a CUDA env struct compiled at run time (promp_b200/_jit.py) into the fused
rollout, env-step and early-termination kernels the built-in envs use.  Everything downstream of the rollout (path table,
sample processing, policy kernels, optimizers, CUDA-graph replay, sharding) takes it unchanged.  See INTEGRATION.md,
"Your own environment", for the struct a user writes.
"""
import numpy as np

from promp_b200 import _jit, _lib
from promp_b200.envs.base import Box, MetaEnv


class CudaEnvProgram(object):
    """The kernels of one env struct: a cubin per requested policy variant (the env-step and env-observe kernels alone for
    hidden=None), compiled (or read from the disk cache) on first request and loaded as a module on first use.  Pickles
    without its modules; they are re-created lazily."""

    def __init__(self, source, struct_name, dims, low, high):
        self.source, self.struct_name, self.dims = source, struct_name, tuple(int(d) for d in dims)
        self.low, self.high = [float(v) for v in low], [float(v) for v in high]
        self._tu = _jit.translation_unit(source, struct_name, self.dims, self.low, self.high)
        self._images, self._handles = {}, {}

    def kernels(self, hidden=None):
        """(cubin, {slot: lowered name}) of a variant; compiles on a cache miss."""
        if hidden not in self._images:
            self._images[hidden] = _jit.compile_kernels(self._tu, _jit.name_expressions(() if hidden is None else (hidden,)))
        return self._images[hidden]

    def handle(self, hidden=None):
        """Loaded module (promp_env_module_load) of a variant."""
        import ctypes
        h = self._handles.get(hidden)
        if h is None:
            image, names = self.kernels(hidden)
            arr = (ctypes.c_char_p * _lib.ENV_MODULE_SLOTS)(*[names.get(i, '').encode() for i in range(_lib.ENV_MODULE_SLOTS)])
            dims = (ctypes.c_int * _lib.ENV_MODULE_NDIMS)(*self.dims)
            out = ctypes.c_void_p()
            _lib.call('promp_env_module_load', image, len(image), ctypes.cast(arr, ctypes.c_void_p), _lib.ENV_MODULE_SLOTS,
                      ctypes.cast(dims, ctypes.c_void_p), ctypes.byref(out))
            h = self._handles[hidden] = out.value
        return h

    def __getstate__(self):
        return dict(source=self.source, struct_name=self.struct_name, dims=self.dims, low=self.low, high=self.high)

    def __setstate__(self, d):
        self.__init__(**d)

    def __del__(self):
        for h in getattr(self, '_handles', {}).values():
            try:
                _lib.load().promp_env_module_unload(h)
            except Exception:     # interpreter shutdown: the library may already be gone
                pass


class CudaMetaEnv(MetaEnv):
    """A MetaEnv whose dynamics are a user's CUDA struct (the serial concept of csrc/user_env.cuh, or any type with the
    built-ins' warp concept, e.g. `promp::Walker`).

    Args:
        cuda_source: source defining the struct `struct_name` (may be empty when struct_name names a built-in type).
        obs_dim, act_dim, state_dim, task_dim: the struct's DO, DA, SD, TD (checked at compile time).
        action_space: Box with the env's action bounds; normalize(env) maps policy actions onto them (scale 10).
        sample_tasks(n) -> list of tasks; task_vector(task) -> float vector [task_dim] the kernels get;
        host_reset_states(n) -> [n, state_dim] reset states from the global numpy RNG in the reference's order
            (reset_mode='numpy').  set_task(task) / get_task(): default keep the task on the env.
        info_keys: names of the env-info channels the struct writes (NINFO = len, at most 3).
        ends_early: the struct's ENDS_EARLY (paths end on `done`: the early-termination kernel and the path table).
        log_diagnostics(paths, prefix): optional.
    Callables must pickle (module-level functions) for snapshots.  The kernels are compiled at construction (compile
    errors raise CudaEnvCompileError with NVRTC's log) and loaded on the device on first use.
    """

    def __init__(self, cuda_source, obs_dim, act_dim, state_dim, task_dim, action_space, sample_tasks, task_vector,
                 host_reset_states, set_task=None, get_task=None, info_keys=(), ends_early=False, log_diagnostics=None,
                 struct_name='UserEnv'):
        self._args = dict(cuda_source=cuda_source, obs_dim=obs_dim, act_dim=act_dim, state_dim=state_dim, task_dim=task_dim,
                          action_space=action_space, sample_tasks=sample_tasks, task_vector=task_vector,
                          host_reset_states=host_reset_states, set_task=set_task, get_task=get_task, info_keys=info_keys,
                          ends_early=ends_early, log_diagnostics=log_diagnostics, struct_name=struct_name)
        self._setup(compile_now=True, **self._args)

    def _setup(self, compile_now, cuda_source, obs_dim, act_dim, state_dim, task_dim, action_space, sample_tasks, task_vector,
               host_reset_states, set_task, get_task, info_keys, ends_early, log_diagnostics, struct_name):
        if not 1 <= int(obs_dim) <= 19:
            raise NotImplementedError("CudaMetaEnv: obs_dim %d; the device policy takes observation sizes 1..19" % obs_dim)
        if not 1 <= int(act_dim) <= 8:
            raise NotImplementedError("CudaMetaEnv: act_dim %d; the device policy takes action sizes 1..8" % act_dim)
        if len(info_keys) > 3:
            raise NotImplementedError("CudaMetaEnv: %d info_keys; the rollout records at most 3 env-info channels"
                                      % len(info_keys))
        if int(state_dim) < 1 or int(task_dim) < 1:
            raise ValueError("CudaMetaEnv: state_dim and task_dim must be >= 1")
        low, high = np.asarray(action_space.low, np.float32).ravel(), np.asarray(action_space.high, np.float32).ravel()
        if low.size != act_dim or high.size != act_dim:
            raise ValueError("CudaMetaEnv: action_space has %d bounds, act_dim is %d" % (low.size, act_dim))
        self.obs_dim, self.act_dim, self.state_dim, self.task_dim = int(obs_dim), int(act_dim), int(state_dim), int(task_dim)
        self.observation_space = Box(-np.inf, np.inf, shape=(self.obs_dim,))
        self.action_space = Box(low, high, dtype=np.float32)
        self.info_keys, self.ends_early = tuple(info_keys), bool(ends_early)
        self._sample_tasks, self._task_vector, self._host_reset_states = sample_tasks, task_vector, host_reset_states
        self._set_task, self._get_task, self._log_diagnostics = set_task, get_task, log_diagnostics
        self._task = None
        dims = (self.obs_dim, self.act_dim, self.state_dim, self.task_dim, len(self.info_keys), int(self.ends_early))
        self.program = CudaEnvProgram(cuda_source, struct_name, dims, low, high)
        if compile_now:
            self.program.kernels()      # a source NVRTC rejects raises here, before anything is launched

    # ---- MetaEnv
    def sample_tasks(self, n_tasks):
        return self._sample_tasks(n_tasks)

    def set_task(self, task):
        self._task = task
        if self._set_task is not None:
            self._set_task(task)

    def get_task(self):
        return self._get_task() if self._get_task is not None else self._task

    def log_diagnostics(self, paths, prefix=''):
        if self._log_diagnostics is not None:
            self._log_diagnostics(paths, prefix)

    def task_vector(self, task):
        return np.asarray(self._task_vector(task), dtype=np.float32).reshape(self.task_dim)

    def host_reset_states(self, n):
        return np.asarray(self._host_reset_states(n), dtype=np.float64).reshape(n, self.state_dim)

    def device_spec(self):
        return dict(env_kind=None, module=self.program, reward_type=self.reward_type, radius=float(self.sparse_reward_radius),
                    obs_dim=self.obs_dim, act_dim=self.act_dim, state_dim=self.state_dim, task_dim=self.task_dim,
                    ends_early=self.ends_early, ninfo=len(self.info_keys))

    # ---- pickling (snapshots, Trainer.restore): the arguments; the modules are re-created on first use
    def __getstate__(self):
        return dict(args=self._args, task=self._task, reward_type=self.reward_type, radius=self.sparse_reward_radius)

    def __setstate__(self, d):
        self._args = d['args']
        self._setup(compile_now=False, **self._args)
        self._task, self.reward_type, self.sparse_reward_radius = d['task'], d['reward_type'], d['radius']
