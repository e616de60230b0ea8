"""promp_set_tasks: the task vectors of a phase travel in the kernel arguments, per task and repeated per env."""
import numpy as np
import pytest

from promp_b200 import _lib


@pytest.mark.gpu
@pytest.mark.parametrize("M,td,E", [(1, 1, 1), (40, 2, 20), (40, 1, 20), (7, 3, 5), (500, 2, 3), (333, 5, 2)])
@pytest.mark.parametrize("with_env", [True, False])
def test_set_tasks_matches_host_broadcast(M, td, E, with_env):
    """Every value lands in place, across the 960-value launch chunks (M * td up to 1665), with and without the per-env
    copy; entries the call does not own stay untouched."""
    import torch
    _lib.require_cuda()
    rng = np.random.RandomState(M * 100 + td * 10 + E)
    vec = rng.standard_normal((M, td)).astype(np.float32)
    per_task = torch.full((M + 1, td), -7.0, device='cuda')
    per_env = torch.full((M * E + 1, td), -7.0, device='cuda')
    _lib.call('promp_set_tasks', M, td, E, vec.ctypes.data, _lib.ptr(per_task), _lib.ptr(per_env) if with_env else None,
              _lib.stream())
    got_t, got_e = per_task.cpu().numpy(), per_env.cpu().numpy()
    assert np.array_equal(got_t[:M], vec)
    assert (got_t[M] == -7.0).all()
    if with_env:
        assert np.array_equal(got_e[:M * E], np.repeat(vec, E, axis=0))
    else:
        assert (got_e[:M * E] == -7.0).all()
    assert (got_e[M * E] == -7.0).all()


@pytest.mark.gpu
def test_set_tasks_host_buffer_reusable_at_once():
    """The values are taken at the call: overwriting the host array right after does not change what lands."""
    import torch
    _lib.require_cuda()
    torch.cuda.synchronize()
    busy = torch.randn(4096, 4096, device='cuda')
    for _ in range(8):
        busy = busy @ busy * 1e-3            # queued work ahead of the call
    vec = np.arange(80, dtype=np.float32).reshape(40, 2)
    per_task = torch.zeros(40, 2, device='cuda')
    per_env = torch.zeros(800, 2, device='cuda')
    _lib.call('promp_set_tasks', 40, 2, 20, vec.ctypes.data, _lib.ptr(per_task), _lib.ptr(per_env), _lib.stream())
    want = vec.copy()
    vec[:] = -1.0
    assert np.array_equal(per_task.cpu().numpy(), want)
    assert np.array_equal(per_env.cpu().numpy(), np.repeat(want, 20, axis=0))


@pytest.mark.gpu
@pytest.mark.parametrize("env_name", ["MetaPointEnvCorner", "HalfCheetahRandDirecEnv"])
def test_executor_set_tasks(env_name):
    """MetaDeviceEnvExecutor.set_tasks leaves the task vectors of the drawn tasks in both device buffers."""
    import torch
    from promp_b200 import envs
    from promp_b200.samplers.vectorized_env_executor import MetaDeviceEnvExecutor
    _lib.require_cuda()
    np.random.seed(3)
    env = envs.normalize(getattr(envs, env_name)())
    ex = MetaDeviceEnvExecutor(env, meta_batch_size=6, envs_per_task=4, max_path_length=10)
    tasks = env.sample_tasks(6)
    ex.set_tasks(tasks)
    inner = getattr(env, '_wrapped_env', env)
    want = np.stack([inner.task_vector(t) for t in tasks]).astype(np.float32).reshape(6, -1)
    torch.cuda.synchronize()
    assert np.array_equal(ex.task_params_per_task.cpu().numpy(), want)
    assert np.array_equal(ex.task_params.cpu().numpy(), np.repeat(want, 4, axis=0))
