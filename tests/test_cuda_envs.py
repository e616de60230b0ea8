"""Users' own environments (promp_b200.envs.CudaMetaEnv): env structs compiled at run time by NVRTC into the fused rollout,
env-step and early-termination kernels.

CPU: the compiler path (sm_90a cubins with every requested kernel, the disk cache, rejections), pickling, host resets.
GPU: the twins of built-in envs against the library's kernels, two example envs against a float64 numpy statement of
their dynamics, sharding, and end-to-end training.
"""
import os
import pickle

import numpy as np
import pytest

from promp_b200 import _jit, _lib
from promp_b200.envs import Box, CudaMetaEnv, normalize

# ---------------------------------------------------------------------------------------------------- example envs
# A damped pendulum: fixed horizon, obs (cos, sin, thd), act 1 (torque, bounds +-2), task = gravity, one info channel.
PENDULUM = r'''
struct Pendulum {
    static constexpr int DO = 3, DA = 1, SD = 2, TD = 1, NINFO = 1;
    static constexpr bool ENDS_EARLY = false;
    static void reset(float (&s)[SD], const float* task, promp::EnvDraw& rng) {
        s[0] = -3.14159265f + 6.2831853f * rng.uniform(0);
        s[1] = -1.f + 2.f * rng.uniform(1);
    }
    static float step(float (&s)[SD], const float* a, const float* task, float* info, int info_stride, bool& done) {
        const float u = fminf(fmaxf(a[0], -2.f), 2.f), th = s[0], thd = s[1];
        const float cost = (1.f - cosf(th)) + 0.1f * thd * thd + 0.001f * u * u;
        const float nthd = thd + 0.05f * (-task[0] * sinf(th) - 0.5f * thd + u);
        s[0] = th + 0.05f * nthd;
        s[1] = nthd;
        info[0] = -0.001f * u * u;
        return -cost;
    }
    static void observe(const float (&s)[SD], float* obs) {
        obs[0] = cosf(s[0]);
        obs[1] = sinf(s[0]);
        obs[2] = s[1];
    }
};
'''


def pendulum_step64(s, a, task):
    u = np.clip(a[..., 0], -2, 2)
    th, thd = s[..., 0], s[..., 1]
    cost = (1 - np.cos(th)) + 0.1 * thd * thd + 0.001 * u * u
    nthd = thd + 0.05 * (-task[..., 0] * np.sin(th) - 0.5 * thd + u)
    return np.stack([th + 0.05 * nthd, nthd], -1), -cost, -0.001 * u * u


def pendulum_obs64(s):
    return np.stack([np.cos(s[..., 0]), np.sin(s[..., 0]), s[..., 1]], -1)


def pendulum_tasks(n):
    return list(np.random.uniform(5.0, 15.0, size=n))


def pendulum_task_vector(task):
    return [task]


def pendulum_resets(n):
    return np.stack([np.random.uniform(-np.pi, np.pi, size=n), np.random.uniform(-1, 1, size=n)], -1)


def make_pendulum():
    return CudaMetaEnv(PENDULUM, obs_dim=3, act_dim=1, state_dim=2, task_dim=1, action_space=Box(-2.0, 2.0, shape=(1,)),
                       sample_tasks=pendulum_tasks, task_vector=pendulum_task_vector, host_reset_states=pendulum_resets,
                       info_keys=('reward_ctrl',), struct_name='Pendulum')


# A gym-style cart-pole whose pole half-length is the task: ends early when the pole falls or the cart leaves the track.
CARTPOLE = r'''
struct CartPole {
    static constexpr int DO = 4, DA = 1, SD = 4, TD = 1, NINFO = 0;
    static constexpr bool ENDS_EARLY = true;
    static void reset(float (&s)[SD], const float*, promp::EnvDraw& rng) {
        for (int i = 0; i < 4; ++i) s[i] = -0.05f + 0.1f * rng.uniform(i);
    }
    static float step(float (&s)[SD], const float* a, const float* task, float*, int, bool& done) {
        const float len = task[0], mp = 0.1f, mt = 1.1f, pml = mp * len;
        const float force = 10.f * fminf(fmaxf(a[0], -1.f), 1.f);
        const float c = cosf(s[2]), sn = sinf(s[2]);
        const float tmp = (force + pml * s[3] * s[3] * sn) / mt;
        const float thacc = (9.8f * sn - c * tmp) / (len * (4.f / 3.f - mp * c * c / mt));
        const float xacc = tmp - pml * thacc * c / mt;
        s[0] = s[0] + 0.02f * s[1];
        s[1] = s[1] + 0.02f * xacc;
        s[2] = s[2] + 0.02f * s[3];
        s[3] = s[3] + 0.02f * thacc;
        done = fabsf(s[0]) > 2.4f || fabsf(s[2]) > 0.20943951f;
        return 1.f;
    }
    static void observe(const float (&s)[SD], float* obs) {
        for (int i = 0; i < 4; ++i) obs[i] = s[i];
    }
};
'''


def cartpole_step64(s, a, task):
    ln = task[..., 0]
    mp, mt = 0.1, 1.1
    pml = mp * ln
    force = 10 * np.clip(a[..., 0], -1, 1)
    c, sn = np.cos(s[..., 2]), np.sin(s[..., 2])
    tmp = (force + pml * s[..., 3] ** 2 * sn) / mt
    thacc = (9.8 * sn - c * tmp) / (ln * (4 / 3 - mp * c * c / mt))
    xacc = tmp - pml * thacc * c / mt
    n = np.stack([s[..., 0] + 0.02 * s[..., 1], s[..., 1] + 0.02 * xacc, s[..., 2] + 0.02 * s[..., 3],
                  s[..., 3] + 0.02 * thacc], -1)
    done = (np.abs(n[..., 0]) > 2.4) | (np.abs(n[..., 2]) > 0.20943951)
    return n, np.ones_like(ln), done


def cartpole_tasks(n):
    return list(np.random.uniform(0.3, 0.8, size=n))


def cartpole_resets(n):
    return np.random.uniform(-0.05, 0.05, size=(n, 4))


def make_cartpole():
    return CudaMetaEnv(CARTPOLE, obs_dim=4, act_dim=1, state_dim=4, task_dim=1, action_space=Box(-1.0, 1.0, shape=(1,)),
                       sample_tasks=cartpole_tasks, task_vector=pendulum_task_vector, host_reset_states=cartpole_resets,
                       ends_early=True, struct_name='CartPole')


def _twin(kind):
    """The built-in env type of `kind` through the expert (warp) concept."""
    from promp_b200.envs import HalfCheetahRandDirecEnv, MetaPointEnvCorner, Walker2DRandVelEnv
    inner = dict(point=MetaPointEnvCorner, cheetah=HalfCheetahRandDirecEnv, walker=Walker2DRandVelEnv)[kind]()
    struct = dict(point='promp::PointCorner', cheetah='promp::Cheetah', walker='promp::Walker')[kind]
    sd, td = dict(point=(2, 2), cheetah=(18, 1), walker=(18, 2))[kind]
    info = ('reward_run', 'reward_ctrl') if kind == 'cheetah' else ()
    return inner, CudaMetaEnv('', obs_dim=inner.obs_dim, act_dim=inner.act_dim, state_dim=sd, task_dim=td,
                              action_space=inner.action_space, sample_tasks=inner.sample_tasks, task_vector=inner.task_vector,
                              host_reset_states=inner.host_reset_states, info_keys=info, ends_early=(kind == 'walker'),
                              struct_name=struct)


@pytest.fixture(autouse=True)
def _jit_cache(tmp_path_factory, monkeypatch):
    # one cache per test session, never the user's
    monkeypatch.setenv('PROMP_B200_JIT_CACHE', str(tmp_path_factory.getbasetemp() / 'jit_cache'))


# ---------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('make', ['point', 'cheetah', 'walker', 'pendulum', 'cartpole'])
def test_compiles_every_kernel(make):
    env = make_pendulum() if make == 'pendulum' else make_cartpole() if make == 'cartpole' else _twin(make)[1]
    hiddens = (64, 32, 64 | _lib.ACT_RELU, 64 | _lib.OUT_TANH, 32 | _lib.ACT_RELU | _lib.OUT_TANH)
    for h in hiddens:
        image, names = env.program.kernels(h)
        assert image[:4] == b'\x7fELF'
        want = {_lib.ENV_SLOT_STEP, _lib.ENV_SLOT_OBSERVE, _jit.rollout_slot(h, False), _jit.rollout_slot(h, True)}
        assert set(names) == want
        for slot, name in names.items():
            assert name.encode() in image, (slot, name)
    # the ELF's machine flags carry the SM: sm_90a cubins say 90 in e_flags' low byte
    assert int.from_bytes(image[48:52], 'little') & 0xff == 90


def test_cache_hit_and_miss():
    make_pendulum().program.kernels(64)
    c0 = dict(_jit.STATS)
    make_pendulum().program.kernels(64)
    assert _jit.STATS['compiles'] == c0['compiles'] and _jit.STATS['cache_hits'] == c0['cache_hits'] + 2
    CudaMetaEnv(PENDULUM.replace('0.5f * thd', '0.25f * thd'), obs_dim=3, act_dim=1, state_dim=2, task_dim=1,
                action_space=Box(-2.0, 2.0, shape=(1,)), sample_tasks=pendulum_tasks, task_vector=pendulum_task_vector,
                host_reset_states=pendulum_resets, info_keys=('reward_ctrl',), struct_name='Pendulum')
    assert _jit.STATS['compiles'] == c0['compiles'] + 1
    assert os.path.realpath(_jit.cache_dir()) != os.path.realpath(os.path.dirname(os.path.dirname(_jit.__file__)))


def _pendulum_with(src, **kw):
    args = dict(obs_dim=3, act_dim=1, state_dim=2, task_dim=1, action_space=Box(-2.0, 2.0, shape=(1,)),
                sample_tasks=pendulum_tasks, task_vector=pendulum_task_vector, host_reset_states=pendulum_resets,
                info_keys=('reward_ctrl',), struct_name='Pendulum')
    args.update(kw)
    return CudaMetaEnv(src, **args)


def test_rejections():
    with pytest.raises(_jit.CudaEnvCompileError) as ei:
        _pendulum_with(PENDULUM.replace('s[1] = nthd;', 's[1] = nthd'))
    assert 'error' in ei.value.log and 'user_env' in ei.value.log
    with pytest.raises(_jit.CudaEnvCompileError) as ei:        # no observe member
        _pendulum_with(PENDULUM[:PENDULUM.index('    static void observe')] + '};\n')
    assert 'observe' in ei.value.log
    with pytest.raises(_jit.CudaEnvCompileError) as ei:        # DO = 20: outside the policy's range
        _pendulum_with(PENDULUM.replace('DO = 3', 'DO = 20'))
    assert 'DO must be 1..19' in ei.value.log
    with pytest.raises(NotImplementedError, match='obs_dim 20'):
        _pendulum_with(PENDULUM.replace('DO = 3', 'DO = 20'), obs_dim=20)
    with pytest.raises(NotImplementedError, match='act_dim 9'):
        _pendulum_with(PENDULUM, act_dim=9, action_space=Box(-2.0, 2.0, shape=(9,)))
    with pytest.raises(NotImplementedError, match='4 info_keys'):
        _pendulum_with(PENDULUM, info_keys=('a', 'b', 'c', 'd'))
    with pytest.raises(_jit.CudaEnvCompileError, match='does not match the declared state_dim'):
        _pendulum_with(PENDULUM, state_dim=3)


def test_pickle_round_trip():
    for env in (make_pendulum(), normalize(make_cartpole())):
        env.set_task(0.5)
        c0 = _jit.STATS['compiles']
        env2 = pickle.loads(pickle.dumps(env))
        assert _jit.STATS['compiles'] == c0        # nothing compiled or loaded until first use
        assert env2.get_task() == 0.5
        assert env2.device_spec()['state_dim'] == env.device_spec()['state_dim']
        assert env2.device_spec().get('normalized') == env.device_spec().get('normalized')
        assert env2.program._handles == {}
        image, names = env2.program.kernels(64)
        assert names == env.program.kernels(64)[1]


def test_host_reset_states_numpy_order():
    env = make_cartpole()
    np.random.seed(3)
    got = env.host_reset_states(5)
    np.random.seed(3)
    want = np.stack([np.random.uniform(-0.05, 0.05, size=4) for _ in range(5)])    # gym's per-env reset order
    np.testing.assert_array_equal(got, want)
    assert env.task_vector(0.5).dtype == np.float32 and env.task_vector(0.5).shape == (1,)


# ---------------------------------------------------------------------------------------------------- GPU
SEED = 1234


def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    _lib.require_cuda()
    torch.cuda.set_device(0)
    return torch


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _policy(torch, env, M, hidden=(64, 64)):
    from promp_b200.policies import MetaGaussianMLPPolicy
    torch.manual_seed(5)
    return MetaGaussianMLPPolicy(name='p', obs_dim=env.obs_dim, action_dim=env.act_dim, meta_batch_size=M, hidden_sizes=hidden)


def _sampler(torch, env, M, E, H, reset_mode='device', shard=None, np_seed=11):
    from promp_b200.samplers import MetaSampler
    np.random.seed(np_seed)
    policy = _policy(torch, env, M)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          reset_mode=reset_mode, seed=SEED, task_shard=shard)
    np.random.seed(np_seed + 1)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    return policy, sampler


def _same(a, b, what):
    """Bit for bit when NVRTC is the library's CUDA version (the twins then compile to the library's code); otherwise
    within the project's 1e-4 bar (round-off of another compiler's schedule)."""
    if _jit.matches_library():
        assert np.array_equal(_bits(a), _bits(b)), what
    else:
        a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
        assert np.abs(a - b).max() <= 1e-4 * max(1.0, np.abs(b).max()), what


def _rollout(torch, entry, first, s, policy, sampler, M, E, H, init=None):
    p = _lib.ptr
    params, stride, clip = policy.sampling_params()
    f = lambda *sh: torch.full(sh, float('nan'), device='cuda')     # noqa: E731
    o = dict(obs=f(M, E, H, s['obs_dim']), act=f(M, E, H, s['act_dim']), mean=f(M, E, H, s['act_dim']), rew=f(M, E, H),
             info=f(3, M, E, H), ls=f(M, s['act_dim']), fs=f(M, E, s['state_dim']),
             done=torch.zeros(M, E, H, dtype=torch.uint8, device='cuda'))
    args = (first, s['reward_type'], s['radius'], 1, M, E, H, policy.hidden_arg, p(params), stride,
            p(sampler.vec_env.task_params_per_task), p(init), None, SEED, 3, None, clip, float(policy.min_log_std),
            p(o['obs']), p(o['act']), p(o['mean']), p(o['rew']), p(o['done']), p(o['info']), p(o['ls']), p(o['fs']),
            _lib.stream())
    _lib.call(entry, *args, *((0,) if entry == 'promp_rollout_module' else ()))
    return {k: v.cpu().numpy() for k, v in o.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['point', 'cheetah'])
def test_twin_rollout_matches_builtin(kind):
    torch = _cuda()
    inner, twin = _twin(kind)
    M, E, H = 40, 20, 100
    policy, sampler = _sampler(torch, normalize(inner), M, E, H)
    s = sampler.spec
    builtin = _rollout(torch, 'promp_rollout', s['env_kind'], s, policy, sampler, M, E, H)
    ts = normalize(twin).device_spec()
    mod = _rollout(torch, 'promp_rollout_module', ts['module'].handle(policy.hidden_arg), s, policy, sampler, M, E, H)
    keys = ['obs', 'act', 'mean', 'rew', 'done', 'ls', 'fs'] + (['info'] if kind == 'cheetah' else [])
    for k in keys:
        b, m = builtin[k], mod[k]
        if k == 'info':
            b, m = b[:2], m[:2]
        _same(m, b, (kind, k, 'bit-identical' if _jit.matches_library() else 'NVRTC %d.%d' % _jit.nvrtc().version))


@pytest.mark.gpu
def test_twin_walker_early_term_and_step_kernels():
    torch = _cuda()
    from promp_b200.envs import Walker2DRandVelEnv
    M, E, H = 40, 20, 200
    inner, twin = _twin('walker')
    outs = []
    for env in (normalize(Walker2DRandVelEnv()), normalize(twin)):
        policy, sampler = _sampler(torch, env, M, E, H)
        paths = sampler.obtain_samples()
        ph = paths.phase
        outs.append({k: getattr(ph, k).cpu().numpy() for k in ('cut', 'n_paths', 'n_valid', 'path_off', 'obs', 'act', 'rew')})
    assert sampler.spec.get('module') is not None and sampler._fused_early_ok()
    for k in outs[0]:
        if k in ('cut', 'n_paths', 'n_valid', 'path_off') and not _jit.matches_library():
            continue     # another compiler's round-off may move a fall by one step
        _same(outs[1][k], outs[0][k], ('walker', k))
    # the single-step kernels against promp_env_step / promp_env_observe on random states and actions
    for kind in ('point', 'cheetah', 'walker'):
        inner, twin = _twin(kind)
        res = []
        for env in (normalize(inner), normalize(twin)):
            from promp_b200.samplers.vectorized_env_executor import MetaDeviceEnvExecutor
            np.random.seed(2)
            ex = MetaDeviceEnvExecutor(env, 8, 16, 50)
            ex.set_tasks(env.sample_tasks(8))
            np.random.seed(3)
            o0 = np.asarray(ex.reset())
            a = np.random.uniform(-12, 12, size=(128, env.act_dim))
            o1, r, d, info = ex.step(a)
            res.append((o0, np.asarray(o1), np.asarray(r), d, [sorted(i.items()) for i in info]))
        for i, what in enumerate(('reset obs', 'obs', 'rew', 'done')):
            _same(res[1][i].astype(np.float32), res[0][i].astype(np.float32), (kind, what))


@pytest.mark.gpu
def test_pendulum_step_and_rollout_against_numpy():
    torch = _cuda()
    env = normalize(make_pendulum())
    # env-step kernel on random states and actions (policy space: the NormalizedEnv map to +-2 applies)
    from promp_b200.samplers.vectorized_env_executor import MetaDeviceEnvExecutor
    n = 512
    ex = MetaDeviceEnvExecutor(env, 4, n // 4, 10 ** 6)
    np.random.seed(4)
    ex.set_tasks(env.sample_tasks(4))
    s0 = np.random.uniform(-3, 3, size=(n, 2)).astype(np.float32)
    ex.state.copy_(torch.from_numpy(s0))
    a = np.random.uniform(-12, 12, size=(n, 1)).astype(np.float32)
    o1, r, d, info = ex.step(a)
    task = ex.task_params.cpu().numpy().astype(np.float64)
    u = np.clip(-2 + (a.astype(np.float64) + 10) * 4 / 20, -2, 2)
    s1, r64, ctrl = pendulum_step64(s0.astype(np.float64), u, task)
    np.testing.assert_allclose(np.asarray(o1), pendulum_obs64(s1), atol=1e-5, rtol=0)
    np.testing.assert_allclose(np.asarray(r), r64, atol=1e-5, rtol=0)
    np.testing.assert_allclose([i['reward_ctrl'] for i in info], ctrl, atol=1e-6, rtol=0)
    assert not np.any(d)
    # the fused rollout: numpy replay of the recorded actions from the recorded initial states
    M, E, H = 40, 20, 100
    policy, sampler = _sampler(torch, env, M, E, H, reset_mode='numpy')
    np.random.seed(21)
    init = pendulum_resets(M * E).astype(np.float32)
    sampler.inject(init_state=init)
    ph = sampler.obtain_samples().phase
    obs, act, rew = (getattr(ph, k).cpu().numpy().reshape(M, E, H, -1).astype(np.float64) for k in ('obs', 'act', 'rew'))
    info = ph.info.cpu().numpy().reshape(1, M, E, H)
    task = sampler.vec_env.task_params_per_task.cpu().numpy().astype(np.float64)[:, None, :]
    # step by step from the recorded states: the upright equilibrium is unstable, so a float64 replay of the whole horizon
    # would amplify float32 round-off exponentially.  The dynamics depend on theta only through its sine and cosine, so
    # the state is recovered from the observation (atan2, thd).
    st = init.reshape(M, E, 2).astype(np.float64)
    np.testing.assert_allclose(obs[:, :, 0], pendulum_obs64(st), atol=1e-6, rtol=0)
    for t in range(H):
        st = np.stack([np.arctan2(obs[:, :, t, 1], obs[:, :, t, 0]), obs[:, :, t, 2]], -1)
        u = np.clip(-2 + (act[:, :, t] + 10) * 4 / 20, -2, 2)
        st, r64, ctrl = pendulum_step64(st, u, task)
        np.testing.assert_allclose(rew[:, :, t, 0], r64, atol=1e-4, rtol=0)
        np.testing.assert_allclose(info[0, :, :, t], ctrl, atol=1e-6, rtol=0)
        if t + 1 < H:
            np.testing.assert_allclose(obs[:, :, t + 1], pendulum_obs64(st), atol=1e-4, rtol=0)
    assert ph.info_keys == ('reward_ctrl',)
    # the recorded means are the policy's at the observations (a (3, 1) policy keeps the zero-padded parameter layout)
    params, stride, clip = policy.sampling_params()
    mean = torch.empty(M, E * H, 1, device='cuda')
    _lib.call(policy.entries['forward'], 3, 1, policy.hidden_arg, M, E * H, _lib.ptr(params), stride,
              _lib.ptr(ph.obs.reshape(M, E * H, 3).contiguous()), _lib.ptr(mean), _lib.stream())
    np.testing.assert_allclose(ph.mean.cpu().numpy().reshape(M, E * H, 1), mean.cpu().numpy(), atol=1e-5, rtol=0)
    assert ph.done.cpu().numpy().reshape(M, E, H)[:, :, -1].all()


@pytest.mark.gpu
def test_cartpole_timelines_path_table_and_resets():
    torch = _cuda()
    from test_paths_finalize import collect_until
    env = normalize(make_cartpole())
    M, E, H = 40, 20, 100
    runs = []
    for _ in range(2):
        policy, sampler = _sampler(torch, env, M, E, H)
        assert sampler._fused_early_ok()
        ph = sampler.obtain_samples().phase
        tl = {k: v.cpu().numpy().astype(np.float64) if v.dtype != torch.uint8 else v.cpu().numpy()
              for k, v in ph.timeline.items() if k != 'ws'}
        runs.append((tl, ph.cut.cpu().numpy(), ph.n_paths.cpu().numpy(), ph.path_off.cpu().numpy()))
    tl, cut, n_paths, path_off = runs[0]
    for a, b in zip(runs[0][1:], runs[1][1:]):
        np.testing.assert_array_equal(a, b)
    for k in tl:
        np.testing.assert_array_equal(_bits(tl[k]), _bits(runs[1][0][k]))      # reset draws reproducible per seed
    task = sampler.vec_env.task_params_per_task.cpu().numpy().astype(np.float64)[:, None, :]
    obs, act, done = tl['obs'], tl['act'], tl['done'].astype(bool)
    T = obs.shape[2]
    assert np.all(np.abs(obs[:, :, 0]) <= 0.05)            # initial resets: U(-0.05, 0.05)^4
    ts = np.zeros((M, E), int)
    for t in range(T - 1):
        u = np.clip(-1 + (act[:, :, t] + 10) * 2 / 20, -1, 1)
        nxt, _, dn = cartpole_step64(obs[:, :, t], u, task)
        ts += 1
        fin = dn | (ts >= H)
        np.testing.assert_array_equal(done[:, :, t], fin, err_msg='t=%d' % t)
        keep = ~fin
        np.testing.assert_allclose(obs[:, :, t + 1][keep], nxt[keep], atol=1e-4, rtol=0)
        assert np.all(np.abs(obs[:, :, t + 1][fin]) <= 0.05)   # in-kernel resets inside their bounds
        ts[fin] = 0
    assert np.all(tl['rew'] == 1.0)
    want = collect_until(done, M * E * H)
    assert cut[0] == want.t_star
    np.testing.assert_array_equal(n_paths, [len(p) for p in want.paths])


@pytest.mark.gpu
@pytest.mark.parametrize('which', ['pendulum', 'cartpole'])
def test_sharding_reproduces_one_process(which):
    torch = _cuda()
    make = make_pendulum if which == 'pendulum' else make_cartpole
    MG, E, H, W = 6, 8, 40, 2
    M = MG // W

    def run(shard, m):
        policy, sampler = _sampler(torch, normalize(make()), m, E, H, shard=shard)
        ph = sampler.obtain_samples().phase
        if which == 'pendulum':
            return {k: getattr(ph, k).cpu().numpy() for k in ('obs', 'act', 'mean', 'rew', 'done', 'info')}
        return {k: v.cpu().numpy() for k, v in ph.timeline.items() if k != 'ws'}

    glob = run(None, MG)
    for r in range(W):
        sh = run((r, W), M)
        for k, v in sh.items():
            g = glob[k]
            g = g[:, r * M:(r + 1) * M] if k == 'info' else g[r * M:(r + 1) * M]
            assert np.array_equal(_bits(v), _bits(g)), (which, r, k)


def _train(torch, tr, tmp_path):
    from promp_b200.utils import logger
    th0 = tr.policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='none')
        tr.train()
        kv = dict(logger.last_dump())
    finally:
        logger.reset()
    assert torch.isfinite(tr.policy.theta).all() and not torch.equal(tr.policy.theta, th0)
    for k in ('LossBefore', 'Step_0-AverageReturn', 'Step_1-AverageReturn'):
        assert np.isfinite(kv[k]), k
    return kv


@pytest.mark.gpu
def test_trainer_promp_pendulum_graph_mode(tmp_path):
    torch = _cuda()
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.samplers import MetaSampleProcessor
    runs = []
    for i in range(2):
        env = normalize(make_pendulum())
        np.random.seed(3)
        policy, sampler = _sampler(torch, env, 4, 5, 50, reset_mode='numpy', np_seed=3)
        proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=4, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=3, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
        tr = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                     num_inner_grad_steps=1, use_cuda_graph=True)
        assert tr.graph_capturable()
        kv = _train(torch, tr, tmp_path / str(i))
        assert tr._graph_step is not None
        runs.append((tr.policy.theta.clone(), kv))
    assert torch.equal(runs[0][0], runs[1][0])
    for k, v in runs[0][1].items():
        if 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert v == runs[1][1][k] or (np.isnan(v) and np.isnan(runs[1][1][k])), k


@pytest.mark.gpu
def test_trainer_trpo_maml_cartpole_device_resets(tmp_path):
    torch = _cuda()
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import TRPOMAML
    from promp_b200.meta_trainer import Trainer
    from promp_b200.samplers import MetaSampleProcessor
    env = normalize(make_cartpole())
    policy, sampler = _sampler(torch, env, 4, 5, 50, reset_mode='device')
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = TRPOMAML(policy=policy, step_size=0.01, inner_lr=0.1, meta_batch_size=4, num_inner_grad_steps=1)
    tr = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3, num_inner_grad_steps=1)
    assert not tr.graph_capturable()
    kv = _train(torch, tr, tmp_path)
    assert abs(kv['MeanKLBefore']) < 1e-6 and 0 < kv['MeanKL'] <= 0.01 and kv['LossAfter'] < kv['LossBefore']
