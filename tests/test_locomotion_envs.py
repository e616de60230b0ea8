"""The MuJoCo-free Walker2d and Swimmer surrogates (Walker2DRandVelEnv, Walker2DRandDirecEnv, SwimmerRandVelEnv).

CPU part: the float64 oracle (oracle/locomotion_surrogates.py) against the reference's observation layout, reward
formulas, done rule and env_infos keys; task draws against the unmodified reference classes (tests/golden/
locomotion_tasks.npz, written by oracle/make_locomotion_golden.py); reset draws; the C ABI's env kinds and dims.
GPU part (pytest -m gpu): the single-step and fused rollout kernels against the oracle, the walker's fused
early-termination sampler against the reference's collect-until-enough rule, and three-iteration Trainer runs.
"""
import os
import pickle

import numpy as np
import pytest

from oracle import locomotion_surrogates as ls

ENVS = ('walker_vel', 'walker_direc', 'swimmer')


def _env_cls(name):
    from promp_b200.envs import Walker2DRandVelEnv, Walker2DRandDirecEnv, SwimmerRandVelEnv
    return {'walker_vel': Walker2DRandVelEnv, 'walker_direc': Walker2DRandDirecEnv, 'swimmer': SwimmerRandVelEnv}[name]


def _glorot_policy(rng, n_in, n_out, hidden=64):
    g = lambda a, b: rng.uniform(-1, 1, (a, b)) * np.sqrt(6.0 / (a + b))
    W = [g(n_in, hidden), g(hidden, hidden), g(hidden, n_out)]
    return lambda o: np.tanh(np.tanh(o @ W[0]) @ W[1]) @ W[2]


def _normalized(a):
    """NormalizedEnv action map onto ctrlrange [-1, 1] (envs/normalized_env.py:109-117)."""
    return np.clip(-1.0 + (a + 10.0) * 2.0 / 20.0, -1.0, 1.0)


# ------------------------------------------------------------------------------------------------ CPU
def test_env_kinds_and_dims():
    from promp_b200 import _lib
    lib = _lib.load()
    assert (_lib.ENV_WALKER, _lib.ENV_SWIMMER) == (5, 6)
    assert lib.promp_env_state_dim(_lib.ENV_WALKER) == 18 and lib.promp_env_task_dim(_lib.ENV_WALKER) == 2
    assert lib.promp_env_state_dim(_lib.ENV_SWIMMER) == 10 and lib.promp_env_task_dim(_lib.ENV_SWIMMER) == 1
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'promp_b200.h')).read()
    assert 'PROMP_ENV_WALKER = 5' in hdr and 'PROMP_ENV_SWIMMER = 6' in hdr
    # the swimmer's (8, 2) policy bucket has caps equal to its logical shape: the rollout kernel's PLayout<8, 2, h> reads
    # the parameters the policy kernels write
    import ctypes
    for h in (32, 64):
        out = (ctypes.c_int * 4)()
        assert lib.promp_policy_layout(8, 2, h, out) == 0
        assert list(out) == [8, 2, h, lib.promp_num_params(8, 2, h)]
    for name in ENVS:
        env = _env_cls(name)()
        assert (env.obs_dim, env.act_dim) == ((8, 2) if name == 'swimmer' else (17, 6))
        assert env.observation_space.shape == (env.obs_dim,) and env.action_space.shape == (env.act_dim,)
        assert np.all(env.action_space.low == -1) and np.all(env.action_space.high == 1)


def test_walker_oracle_obs_reward_done():
    rng = np.random.RandomState(0)
    n = 64
    st = ls.walker_reset_state(rng, n)
    qpos, qvel = st[:, :9], st[:, 9:]
    assert np.all(np.abs(qpos[:, 1] - 1.25) <= 0.005) and np.all(np.abs(np.delete(qpos, 1, axis=1)) <= 0.005)
    assert np.all(np.abs(qvel) <= 0.005)
    qvel = qvel.copy()
    qvel[:, 4] = 25.0
    qvel[:, 7] = -13.0
    obs = ls.walker_obs(qpos, qvel)
    assert obs.shape == (n, 17)
    np.testing.assert_array_equal(obs[:, :8], qpos[:, 1:])
    np.testing.assert_array_equal(obs[:, 8:], np.clip(qvel, -10, 10))
    assert np.all(obs[:, 12] == 10.0) and np.all(obs[:, 15] == -10.0)
    u = rng.uniform(-1, 1, (n, 6))
    goal = rng.uniform(0, 10, n)
    q1, v1, r_vel, d, fwd = ls.walker_step(qpos, qvel, u, goal, 1)
    np.testing.assert_allclose(fwd, (q1[:, 0] - qpos[:, 0]) / 0.016, rtol=1e-12)
    np.testing.assert_allclose(r_vel, -np.abs(fwd - goal) + 15.0 - 1e-3 * np.sum(u ** 2, 1), rtol=1e-12)
    direction = rng.choice((-1.0, 1.0), n)
    _, _, r_dir, _, fwd2 = ls.walker_step(qpos, qvel, u, direction, 0)
    np.testing.assert_array_equal(fwd, fwd2)
    np.testing.assert_allclose(r_dir, direction * fwd + 1.0 - 1e-3 * np.sum(u ** 2, 1), rtol=1e-12)
    # done = not (0.8 < z < 2.0 and -1 < angle < 1)
    z = np.array([1.25, 0.8, 0.81, 1.99, 2.0, 0.5, 1.25, 1.25, 1.25, 1.25])
    a = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.99, -0.99, 1.0, -1.0])
    q = np.zeros((10, 9))
    q[:, 1], q[:, 2] = z, a
    np.testing.assert_array_equal(ls.walker_done(q), [False, True, False, False, True, True, False, False, True, True])


def test_walker_random_policy_falls_within_the_horizon():
    """The done rule fires in practice: under normalize(env) a randomly initialised policy with the default action noise
    (log_std 0) falls within H = 200 steps on a good share of paths, so the early-termination path gets exercised."""
    rng = np.random.RandomState(1)
    n, H = 300, 200
    st = ls.walker_reset_state(rng, n)
    qpos, qvel = st[:, :9], st[:, 9:]
    pol = _glorot_policy(rng, 17, 6)
    fell_at = np.full(n, -1)
    for t in range(H):
        a = pol(ls.walker_obs(qpos, qvel)) + rng.randn(n, 6)
        qpos, qvel, _, done, _ = ls.walker_step(qpos, qvel, _normalized(a), 1.0, 0)
        fell_at[(fell_at < 0) & done] = t
    frac = float((fell_at >= 0).mean())
    assert 0.3 <= frac <= 0.95, frac
    assert len(np.unique(fell_at[fell_at >= 0])) > 20          # very different path lengths


def test_swimmer_oracle_obs_reward_info():
    from promp_b200.envs import SwimmerRandVelEnv
    assert 'rewards deviating from the goal' in SwimmerRandVelEnv.__doc__       # the reference's sign quirk is documented
    rng = np.random.RandomState(2)
    n = 32
    st = ls.swimmer_reset_state(rng, n)
    assert np.all(np.abs(st) <= 0.1)
    qpos, qvel = st[:, :5], st[:, 5:]
    obs = ls.swimmer_obs(qpos, qvel)
    assert obs.shape == (n, 8)
    np.testing.assert_array_equal(obs, np.concatenate([qpos[:, 2:], qvel], 1))
    u = rng.uniform(-1, 1, (n, 2))
    goal = rng.uniform(0.1, 0.2, n)
    q1, v1, r, rf, rc = ls.swimmer_step(qpos, qvel, u, goal)
    fwd = (q1[:, 0] - qpos[:, 0]) / 0.04
    np.testing.assert_allclose(rf, np.abs(fwd - goal), rtol=1e-12)      # the reference's sign: |v - goal|, not -|v - goal|
    np.testing.assert_allclose(rc, -1e-4 * np.sum(u ** 2, 1), rtol=1e-12)
    np.testing.assert_allclose(r, rf + rc, rtol=1e-12)
    # a phase-lagged stroke swims forward, its mirror image backward
    t = np.arange(300) * 0.04
    for sgn in (1.0, -1.0):
        qp, qv = np.zeros((1, 5)), np.zeros((1, 5))
        for k in range(300):
            qp, qv, _, _, _ = ls.swimmer_step(qp, qv, np.array([[np.sin(3 * t[k]), sgn * np.cos(3 * t[k])]]), 0.15)
        assert sgn * qp[0, 0] < -1.0 or sgn * qp[0, 0] > 1.0


@pytest.mark.parametrize('name', ENVS)
def test_task_draws_match_reference(name, golden_dir):
    g = np.load(os.path.join(golden_dir, 'locomotion_tasks.npz'))
    cls = _env_cls(name)
    env = cls()
    for seed in (0, 7, 123):
        for n in (1, 5, 40):
            key = '%s_s%d_n%d' % (cls.__name__, seed, n)
            np.random.seed(seed)
            np.testing.assert_array_equal(np.asarray(env.sample_tasks(n), dtype=np.float64), g[key])
            np.testing.assert_array_equal(np.random.uniform(size=3), g[key + '_probe'])
    # construction draws one task like the reference's __init__ (set_task(sample_tasks(1)[0]))
    np.random.seed(7)
    env = cls()
    assert env.get_task() == g['%s_s7_n1' % cls.__name__][0]
    np.testing.assert_array_equal(np.random.uniform(size=3), g['%s_s7_n1_probe' % cls.__name__])
    assert cls(0.5).get_task() == 0.5
    env.set_task(0.25)
    assert env.get_task() == 0.25
    tv = env.task_vector(0.25)
    assert tv.dtype == np.float32 and tv[0] == 0.25
    if name.startswith('walker'):
        assert list(tv) == [0.25, 1.0 if name == 'walker_vel' else 0.0]


@pytest.mark.parametrize('name', ENVS)
def test_host_reset_draws(name):
    env = _env_cls(name)()
    np.random.seed(3)
    got = env.host_reset_states(17)
    np.random.seed(3)
    want = (ls.swimmer_reset_state if name == 'swimmer' else ls.walker_reset_state)(np.random, 17)
    np.testing.assert_array_equal(got, want)
    # exactly 17 * state_dim uniforms consumed: every qpos draw, then every qvel draw
    np.random.seed(3)
    np.random.uniform(size=17 * got.shape[1])
    probe = np.random.uniform(size=2)
    np.random.seed(3)
    env.host_reset_states(17)
    np.testing.assert_array_equal(np.random.uniform(size=2), probe)


@pytest.mark.parametrize('name', ENVS)
def test_pickle_normalize_and_log_diagnostics(name):
    from promp_b200.envs import normalize
    from promp_b200.utils import logger
    env = normalize(_env_cls(name)(0.15))
    assert np.all(env.action_space.high == 10.0)
    env2 = pickle.loads(pickle.dumps(env))
    assert type(env2._wrapped_env) is type(env._wrapped_env) and env2.get_task() == 0.15
    rng = np.random.RandomState(0)
    paths = [dict(observations=rng.randn(L, env.obs_dim), env_infos={}) for L in (5, 9)]
    logger.set_quiet(True)
    logger.reset()
    env.log_diagnostics(paths, prefix='p-')
    kv = dict(logger.getkvs())
    if name == 'swimmer':
        progs = [p['observations'][-1][-3] - p['observations'][0][-3] for p in paths]
        assert kv['p-AverageForwardProgress'] == np.mean(progs) and kv['p-StdForwardProgress'] == np.std(progs)
        assert kv['p-MaxForwardProgress'] == np.max(progs) and kv['p-MinForwardProgress'] == np.min(progs)
        assert env.info_keys == ('reward_fwd', 'reward_ctrl')
    else:
        assert not any(k.startswith('p-') for k in kv) and env.info_keys == ()
    logger.reset()


# ------------------------------------------------------------------------------------------------ GPU
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _oracle_step(name, st, u, task):
    """float64 oracle step on [n, state_dim] states -> (state', reward, done, info rows)."""
    nq = st.shape[1] // 2
    qpos, qvel = st[:, :nq], st[:, nq:]
    if name == 'swimmer':
        q, v, r, rf, rc = ls.swimmer_step(qpos, qvel, u, task)
        return np.concatenate([q, v], 1), r, np.zeros(len(r), bool), (rf, rc)
    q, v, r, d, _ = ls.walker_step(qpos, qvel, u, task, 1 if name == 'walker_vel' else 0)
    return np.concatenate([q, v], 1), r, d, ()


def _obs(name, st):
    nq = st.shape[1] // 2
    return (ls.swimmer_obs if name == 'swimmer' else ls.walker_obs)(st[..., :nq], st[..., nq:])


def _near_threshold(st):
    z, a = st[:, 1], st[:, 2]
    return np.minimum.reduce([np.abs(z - 0.8), np.abs(z - 2.0), np.abs(np.abs(a) - 1.0)]) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize('name', ENVS)
def test_env_step_kernel_matches_oracle(name):
    """promp_env_step vs the float64 oracle, step by step for 150 steps from shared states with fed actions (the device
    state is glued to the oracle every step).  Walker: the states drift from standing to fallen, so both sides of the
    done rule are visited; flags differ only within float32 round-off of a threshold."""
    torch = _cuda()
    from promp_b200.envs import normalize
    from promp_b200.samplers import MetaDeviceEnvExecutor
    n, T = 96, 150
    rng = np.random.RandomState(4)
    env = normalize(_env_cls(name)())
    tasks = list(env.sample_tasks(n))
    ex = MetaDeviceEnvExecutor(env, n, 1, max_path_length=10 ** 6)
    ex.set_tasks(tasks)
    task = np.asarray(tasks, dtype=np.float32).astype(np.float64)
    st = (ls.swimmer_reset_state if name == 'swimmer' else ls.walker_reset_state)(rng, n)
    act = 4.0 * rng.randn(T, n, env.act_dim)
    act[::9] *= 4.0                                  # exercise the action clip
    n_flip, n_done = 0, 0
    for t in range(T):
        st32 = st.astype(np.float32)
        st32[:, 0] = 0.0                             # x is not observed and does not feed back: keep it small
        ex.state.copy_(torch.from_numpy(st32))
        ex.ts.zero_()
        a32 = act[t].astype(np.float32)
        obs, rew, dones, infos = ex.step(a32)
        want_st, want_r, want_d, want_info = _oracle_step(name, st32.astype(np.float64), _normalized(a32.astype(np.float64)), task)
        np.testing.assert_allclose(np.asarray(rew), want_r, rtol=1e-5, atol=1e-5)
        flip = dones != want_d
        if name.startswith('walker'):
            assert np.all(_near_threshold(want_st)[flip]), t
        else:
            assert not dones.any()
        n_flip += int(flip.sum())
        n_done += int(want_d.sum())
        keep = ~(dones | want_d)                     # a done env is reset with fresh host draws
        np.testing.assert_allclose(np.asarray(obs)[keep], _obs(name, want_st)[keep], rtol=1e-5, atol=2e-5)
        if name == 'swimmer':
            assert set(infos[0]) == {'reward_fwd', 'reward_ctrl'}
            np.testing.assert_allclose([i['reward_fwd'] for i in infos], want_info[0], rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose([i['reward_ctrl'] for i in infos], want_info[1], rtol=1e-5, atol=1e-9)
        else:
            assert infos[0] == {}
        st = want_st
    assert n_flip <= 2, n_flip
    if name.startswith('walker'):
        assert n_done > n, n_done                    # the done rule fired


def _stack(name, M, E, H, hidden=64, seed=3, **kw):
    from promp_b200.envs import normalize
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler
    np.random.seed(seed)
    env = normalize(_env_cls(name)())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=env.obs_dim, action_dim=env.act_dim, meta_batch_size=M,
                                   hidden_sizes=(hidden, hidden))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H, **kw)
    return env, policy, sampler


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', [64, 32])
@pytest.mark.parametrize('name', ENVS)
def test_fused_rollout_matches_oracle(name, hidden):
    """promp_rollout with fed noise and init states vs the oracle: the policy mean against the float64 policy on the
    kernel's observations, a = mean + eps*exp(log_std), and the env trajectory replayed in float64 with the kernel's
    actions (walker: a fixed-horizon record, the fall rule is not applied in promp_rollout)."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.samplers.device_data import PhaseData
    M, E, H = 3, 5, 48
    env, policy, sampler = _stack(name, M, E, H, hidden=hidden)
    sampler.update_tasks()
    Do, Da = env.obs_dim, env.act_dim
    rng = np.random.RandomState(6)
    theta = policy.theta.cpu().numpy()
    theta_tasks = np.stack([theta + 0.05 * rng.randn(theta.size).astype(np.float32) for _ in range(M)])
    policy.update_task_parameters(torch.from_numpy(theta_tasks).cuda())
    noise = rng.randn(M, E, H, Da).astype(np.float32)
    init = (ls.swimmer_reset_state if name == 'swimmer' else ls.walker_reset_state)(rng, M * E).astype(np.float32)
    phase = PhaseData(M, E, H, Do, Da, sampler.device)
    sampler.rollout_into(phase, torch.from_numpy(init.reshape(M, E, -1)).cuda(), torch.from_numpy(noise).cuda())
    obs = phase.obs.cpu().numpy().reshape(M, E, H, Do)
    act = phase.act.cpu().numpy().reshape(M, E, H, Da)
    mean = phase.mean.cpu().numpy().reshape(M, E, H, Da)
    rew = phase.rew.cpu().numpy().reshape(M, E, H)
    done = phase.done.cpu().numpy().reshape(M, E, H)
    assert done[..., :-1].sum() == 0 and (done[..., -1] == 1).all()
    mu, _ = th.dist_info(torch.from_numpy(theta_tasks).double(), torch.from_numpy(obs.reshape(M, E * H, Do)).double(),
                         (Do, Da, (hidden, hidden)))
    np.testing.assert_allclose(mean.reshape(M, E * H, Da), mu.numpy(), rtol=1e-4, atol=2e-5)
    sig = np.exp(theta_tasks[:, -Da:].astype(np.float64))[:, None, None, :]
    np.testing.assert_allclose(act, mean + noise * sig, rtol=1e-5, atol=1e-5)
    task = sampler.vec_env.task_params_per_task.cpu().numpy()[:, 0].astype(np.float64)
    task = np.repeat(task, E)
    st = init.astype(np.float64)
    np.testing.assert_array_equal(obs[:, :, 0].reshape(M * E, Do), _obs(name, init))
    info = phase.info.cpu().numpy().reshape(2, M * E, H) if name == 'swimmer' else None
    if name == 'swimmer':
        assert phase.info_keys == ('reward_fwd', 'reward_ctrl')
    for t in range(H):
        st, r, _, inf = _oracle_step(name, st, _normalized(act[:, :, t].reshape(M * E, Da).astype(np.float64)), task)
        np.testing.assert_allclose(rew[:, :, t].reshape(-1), r, rtol=1e-4, atol=1e-4)
        if name == 'swimmer':
            np.testing.assert_allclose(info[0, :, t], inf[0], rtol=1e-4, atol=1e-4)
            np.testing.assert_allclose(info[1, :, t], inf[1], rtol=1e-4, atol=1e-8)
        if t + 1 < H:
            np.testing.assert_allclose(obs[:, :, t + 1].reshape(M * E, Do), _obs(name, st), rtol=1e-4, atol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['walker_vel', 'walker_direc'])
def test_walker_fused_early_termination(name):
    """reset_mode='device': promp_rollout_early_term records per-slot timelines (paths end when the walker falls or at
    the horizon, slots reset in-kernel) and promp_paths_finalize builds the path table.  Timelines are checked step by
    step against the oracle; the path table and compacted tensors against the reference's collect-until-enough rule on
    the same timelines; the ragged phase then goes through promp_process_samples_ragged and a ProMP step."""
    torch = _cuda()
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.samplers.device_data import DeviceRaggedPhaseData
    M, E, H = 3, 8, 100
    env, policy, sampler = _stack(name, M, E, H, reset_mode='device', seed=4)
    assert sampler._fused_early_ok() and not sampler._fused_ok()
    theta = policy.theta.cpu().numpy().copy()
    # action noise std 10 in policy space (torque std ~1 after normalize) and a mean torque that leans the torso forward:
    # most paths fall after 70-100 steps, at different steps, the rest reach the horizon
    theta[-6:] = np.log(10.0)
    theta[-12:-6] = 2.0 * np.sign(ls.Walker.P)
    policy.set_params(theta)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    paths = sampler.obtain_samples()
    ph = paths.phase
    assert isinstance(ph, DeviceRaggedPhaseData)
    tl = ph.timeline
    T = 2 * H - 1
    done = tl['done'].cpu().numpy().astype(bool)
    t_obs, t_act, t_rew = (tl[k].cpu().numpy().astype(np.float64) for k in ('obs', 'act', 'rew'))
    task = sampler.vec_env.task_params_per_task.cpu().numpy()[:, 0].astype(np.float64)
    mode = 1 if name == 'walker_vel' else 0
    # ---- timelines against the oracle (state rebuilt from the observation: x does not feed back, |qvel| < 10 here)
    assert np.abs(t_obs[..., 8:]).max() < 10.0
    n_fall, n_flip = 0, 0
    for m in range(M):
        st = np.concatenate([np.zeros((E, T, 1)), t_obs[m]], axis=-1)           # [E, T, 18]
        q1, v1, r, d, _ = ls.walker_step(st[..., :9], st[..., 9:], _normalized(t_act[m]), task[m], mode)
        np.testing.assert_allclose(t_rew[m], r, rtol=1e-4, atol=1e-4)
        ts = np.zeros(E, dtype=int)
        for t in range(T):
            ts += 1
            want = d[:, t] | (ts >= H)
            flip = want != done[m, :, t]
            assert np.all(_near_threshold(np.concatenate([q1[:, t], v1[:, t]], 1))[flip]), (m, t)
            n_flip += int(flip.sum())
            n_fall += int((d[:, t] & done[m, :, t]).sum())
            if t + 1 < T:
                for e in range(E):
                    if done[m, e, t]:                # fresh in-kernel reset: init_qpos + U(-.005,.005)
                        nxt = t_obs[m, e, t + 1] - np.r_[1.25, np.zeros(16)]
                        assert np.abs(nxt).max() <= 0.005 + 1e-6
                    else:
                        np.testing.assert_allclose(t_obs[m, e, t + 1], ls.walker_obs(q1[e, t], v1[e, t]), rtol=1e-4, atol=1e-4)
            ts[done[m, :, t]] = 0
    assert n_flip <= 2 and n_fall >= M * E, (n_flip, n_fall)
    # ---- the path table equals the reference rule applied to the same timelines
    from test_paths_finalize import collect_until
    rule = collect_until(done, M * E * H)
    assert rule.reached
    want_paths, t_star = rule.paths, rule.t_star
    cut = ph.cut.cpu().numpy()
    assert cut[0] == t_star and cut[1] == 1
    n_paths, n_valid, off = ph.n_paths_host, ph.n_valid_host, ph.path_off_host
    obs_r, act_r, rew_r, done_r = ph.obs.cpu().numpy(), ph.act.cpu().numpy(), ph.rew.cpu().numpy(), ph.done.cpu().numpy()
    lens = []
    for m in range(M):
        assert n_paths[m] == len(want_paths[m]) and n_valid[m] == sum(p[2] for p in want_paths[m])
        pos = 0
        for k, (e, s0, L) in enumerate(want_paths[m]):
            assert off[m, k] == pos and off[m, k + 1] == pos + L
            np.testing.assert_array_equal(obs_r[m, pos:pos + L], t_obs[m, e, s0:s0 + L].astype(np.float32))
            np.testing.assert_array_equal(act_r[m, pos:pos + L], t_act[m, e, s0:s0 + L].astype(np.float32))
            np.testing.assert_array_equal(rew_r[m, pos:pos + L], t_rew[m, e, s0:s0 + L].astype(np.float32))
            assert done_r[m, pos + L - 1] == 1 and done_r[m, pos:pos + L - 1].sum() == 0
            pos += L
            lens.append(L)
        assert len(paths[m]) == len(want_paths[m])
    assert min(lens) < H and len(set(lens)) > 5              # ragged: paths of many different lengths
    # ---- the ragged phase through the processing kernel and one ProMP step
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    samples = proc.process_samples(paths, log='all', log_prefix='x-')
    adv = ph.adv.cpu().numpy()
    for m in range(M):
        a = adv[m, :n_valid[m]]
        assert np.isfinite(a).all() and abs(a.mean()) < 1e-4 and abs(a.std() - 1) < 1e-3
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=2,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    algo._adapt(samples)
    samples2 = proc.process_samples(sampler.obtain_samples())
    algo.optimize_policy([samples, samples2], log=False)
    assert torch.isfinite(policy.theta).all() and np.isfinite(algo.last_stats['loss_after'])


def _train(name, algo_name, reset_mode, tmp_path, seed):
    import torch
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP, TRPOMAML, VPGMAML
    from promp_b200.meta_trainer import Trainer
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.utils import logger
    M, E, H = 4, 3, 30
    torch.manual_seed(seed)           # the step loop's action noise (MetaGaussianMLPPolicy.get_actions) comes from torch
    env, policy, sampler = _stack(name, M, E, H, seed=seed, reset_mode=reset_mode)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    if algo_name == 'promp':
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=3, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=True)
    elif algo_name == 'trpo':
        algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, step_size=0.01)
    else:
        algo = VPGMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                      num_inner_grad_steps=1)
    theta0 = policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='none')
        trainer.train()
        kv = logger.last_dump()
    finally:
        logger.reset()
    assert not torch.equal(policy.theta, theta0) and torch.isfinite(policy.theta).all()
    return env, policy, trainer, kv


@pytest.mark.gpu
@pytest.mark.parametrize('algo_name', ['promp', 'trpo', 'vpg'])
@pytest.mark.parametrize('name,reset_mode', [('walker_vel', 'numpy'), ('walker_direc', 'numpy'), ('swimmer', 'numpy'),
                                             ('walker_vel', 'device'), ('walker_direc', 'device')])
def test_trainer_runs(name, reset_mode, algo_name, tmp_path):
    """Three meta-iterations through Trainer.train(): finite logged scalars, CUDA-graph mode where the configuration
    allows it (fixed-horizon swimmer with ProMP / TRPO-MAML), identical results for the same seed, env pickle round trip."""
    torch = _cuda()
    env, policy, trainer, kv = _train(name, algo_name, reset_mode, tmp_path / 'a', seed=11)
    _, policy2, _, kv2 = _train(name, algo_name, reset_mode, tmp_path / 'b', seed=11)
    assert kv['Itr'] == 2
    for key in ('Step_0-AverageReturn', 'Step_1-AverageReturn', 'Step_0-AveragePolicyStd', 'Step_1-NumTrajs', 'LossBefore',
                'LossAfter'):
        assert key in kv and np.isfinite(kv[key]), key
    # graph replays log the per-span timer columns as NaN (not separable inside one graph); every other scalar is finite
    assert all(np.isfinite(v) for k, v in kv.items() if isinstance(v, (float, int, np.floating)) and 'Time' not in k)
    if name == 'swimmer':
        assert np.isfinite(kv['Step_1-AverageForwardProgress']) and np.isfinite(kv['Step_0-StdForwardProgress'])
        if algo_name in ('promp', 'trpo'):
            assert trainer.graph_capturable()
    else:
        assert not trainer.graph_capturable()
        assert kv['Step_0-NumTrajs'] >= 4 * 3              # collect-until-enough: at least one path per env slot
    assert torch.equal(policy.theta, policy2.theta)
    for k, v in kv.items():
        if k.startswith('Step_') and 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert v == kv2[k] or (np.isnan(v) and np.isnan(kv2[k])), k
    env2 = pickle.loads(pickle.dumps(env))
    assert type(env2._wrapped_env) is type(env._wrapped_env) and env2.get_task() == env.get_task()
    assert env2.device_spec() == env.device_spec()
