"""GPU parity tests: the CUDA path (through the C ABI, via the reference-shaped Python classes)
against the CPU oracle and the committed golden vectors of the unmodified reference.

Tolerances: integer / index work bit-exact; float32 quantities within 1e-4 relative (the north-star
bar), tighter where the arithmetic allows.  Run on an H100: pytest -m gpu.
"""
import math
import os
from collections import OrderedDict

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


# ------------------------------------------------------------------------------------------------
def _make_stack(env_name, M, E, H, hidden=64, seed=3, **sampler_kw):
    torch = _cuda()
    from promp_b200.envs import normalize, MetaPointEnvCorner, HalfCheetahRandDirecEnv
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    np.random.seed(seed)
    env = normalize(MetaPointEnvCorner() if env_name == 'point' else HalfCheetahRandDirecEnv())
    policy = MetaGaussianMLPPolicy(name="meta-policy", obs_dim=int(np.prod(env.observation_space.shape)),
                                   action_dim=int(np.prod(env.action_space.shape)), meta_batch_size=M,
                                   hidden_sizes=(hidden, hidden))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          **sampler_kw)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    return env, policy, sampler, proc


def test_rollout_matches_reference_golden(golden_dir):
    """configs[0] (M=5,E=4,H=100, seed 1): tasks / reset states / rollouts vs the UNMODIFIED reference
    MetaSampler + normalize(MetaPointEnvCorner) (fixture sampler_rollout.npz), same theta and noise."""
    torch = _cuda()
    g = _load(golden_dir, 'sampler_rollout.npz')
    M, E, H = 5, 4, 100
    env, policy, sampler, proc = _make_stack('point', M, E, H)
    policy.set_params(g['theta'])
    np.random.seed(1)
    for it in range(2):
        sampler.update_tasks()
        goals = sampler.vec_env.task_params_per_task.cpu().numpy()
        assert np.array_equal(goals.astype(np.float64), g['it%d_goals' % it])      # bit-exact task draw
        policy.switch_to_pre_update()
        noise = np.ascontiguousarray(np.transpose(g['noise'][it], (1, 2, 0, 3)))   # [H,M,E,Da] -> [M,E,H,Da]
        sampler.inject(noise=noise)
        paths = sampler.obtain_samples()
        assert list(paths.keys()) == list(range(M)) and all(len(v) == E for v in paths.values())
        obs = np.stack([np.stack([p['observations'] for p in paths[m]]) for m in range(M)])
        act = np.stack([np.stack([p['actions'] for p in paths[m]]) for m in range(M)])
        rew = np.stack([np.stack([p['rewards'] for p in paths[m]]) for m in range(M)])
        mean = np.stack([np.stack([p['agent_infos']['mean'] for p in paths[m]]) for m in range(M)])
        assert obs.shape == (M, E, H, 2)
        # reset states: same numpy draws, float32-rounded
        np.testing.assert_array_equal(obs[:, :, 0], g['it%d_obs' % it][:, :, 0].astype(np.float32))
        np.testing.assert_allclose(obs, g['it%d_obs' % it], rtol=0, atol=2e-5)
        np.testing.assert_allclose(act, g['it%d_act' % it], rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(mean, g['it%d_mean' % it], rtol=1e-4, atol=2e-5)
        # the sparse reward is discontinuous (point_env_2d_corner.py:68-76): a float32 state may fall on the other side of a
        # branch boundary.  Every mismatch must sit ON such a boundary of the reference state s' (L1 radius 0.5, or a
        # nearest-corner tie x = 0 / y = 0), and there may be at most 3 of them in 2 000 samples.
        bad = np.abs(rew - g['it%d_rew' % it]) > 1e-4
        assert bad.sum() <= 3, int(bad.sum())
        ref_obs = g['it%d_obs' % it]
        for m_, e_, t_ in zip(*np.nonzero(bad)):
            if t_ + 1 < H:
                x, y = ref_obs[m_, e_, t_ + 1]
                margin = min(abs(abs(x) + abs(y) - 0.5), abs(x), abs(y))
                assert margin < 1e-3, (m_, e_, t_, x, y)
    # the numpy stream was consumed exactly like the reference consumed it
    assert np.array_equal(np.random.uniform(size=4), g['rng_probe_after'])


def test_env_step_kernel_matches_reference_golden(golden_dir):
    """promp_env_step (vec-env API) vs the reference envs for all three reward types + early-done PointEnv."""
    torch = _cuda()
    from promp_b200.envs import normalize, MetaPointEnvCorner, MetaPointEnv
    from promp_b200.samplers import MetaDeviceEnvExecutor
    g = _load(golden_dir, 'point_corner_steps.npz')
    T, n_env, _ = g['actions'].shape
    for rtype in ('sparse', 'dense', 'dense_squared'):
        ex = MetaDeviceEnvExecutor(normalize(MetaPointEnvCorner(reward_type=rtype)), n_env, 1, max_path_length=10 ** 6)
        ex.set_tasks(list(g['goals']))
        ex.state.copy_(torch.from_numpy(g['obs0'].astype(np.float32)))
        n_bad = 0
        for t in range(T):
            obs, rew, dones, infos = ex.step(g['actions'][t])
            np.testing.assert_allclose(np.asarray(obs), g['next_obs_' + rtype][t], rtol=0, atol=5e-5)
            n_bad += int((np.abs(np.asarray(rew) - g['rewards_' + rtype][t]) > 1e-4).sum())
            assert not dones.any() and infos[0] == {}
            # keep the device trajectory glued to the reference so float32 drift cannot accumulate
            ex.state.copy_(torch.from_numpy(g['next_obs_' + rtype][t].astype(np.float32)))
        assert n_bad <= (3 if rtype == 'sparse' else 0), (rtype, n_bad)
    g = _load(golden_dir, 'point_env_steps.npz')
    T, n_env, _ = g['actions'].shape
    np.random.seed(0)
    ex = MetaDeviceEnvExecutor(normalize(MetaPointEnv()), n_env, 1, max_path_length=10 ** 6)
    ex.set_tasks([{}] * n_env)
    ex.state.copy_(torch.from_numpy(g['obs0'].astype(np.float32)))
    for t in range(T):
        st_before = ex.state.cpu().numpy().copy()
        obs, rew, dones, _ = ex.step(g['actions'][t])
        np.testing.assert_allclose(np.asarray(rew), g['rewards'][t], rtol=1e-4, atol=1e-5)
        assert np.array_equal(dones, g['dones'][t]) or np.abs(np.abs(g['next_obs'][t]) - 0.01).min() < 1e-5
        ex.state.copy_(torch.from_numpy(g['next_obs'][t].astype(np.float32)))
        ex.ts.zero_()


@pytest.mark.parametrize('env_name,M,E,H,hidden', [('point', 4, 5, 70, 64), ('cheetah', 3, 4, 45, 64),
                                                    ('cheetah', 2, 3, 40, 32), ('point', 2, 3, 33, 32)])
def test_rollout_teacher_forced_vs_oracle(env_name, M, E, H, hidden):
    """Fused rollout vs the CPU oracle: policy forward on the kernel's own observations, sampling rule,
    and env transitions replayed with the kernel's own actions (removes closed-loop drift)."""
    torch = _cuda()
    from oracle import tf_half as th, numpy_half as nh, cheetah_surrogate as cs
    env, policy, sampler, proc = _make_stack(env_name, M, E, H, hidden=hidden)
    sampler.update_tasks()
    Do, Da = policy.obs_dim, policy.action_dim
    rng = np.random.RandomState(5)
    noise = rng.randn(M, E, H, Da).astype(np.float32)
    # post-update style per-task parameters to exercise param_stride != 0
    theta = policy.theta.cpu().numpy()
    theta_tasks = np.stack([theta + 0.05 * rng.randn(theta.size).astype(np.float32) for _ in range(M)])
    policy.update_task_parameters(torch.from_numpy(theta_tasks).cuda())
    sampler.inject(noise=noise)
    paths = sampler.obtain_samples()
    ph = paths.phase
    obs = ph.obs.cpu().numpy().reshape(M, E, H, Do)
    act = ph.act.cpu().numpy().reshape(M, E, H, Da)
    mean = ph.mean.cpu().numpy().reshape(M, E, H, Da)
    rew = ph.rew.cpu().numpy().reshape(M, E, H)
    done = ph.done.cpu().numpy().reshape(M, E, H)
    assert done[..., :-1].sum() == 0 and (done[..., -1] == 1).all()
    # (1) policy forward (float32 oracle) on the kernel's observations
    mu_o, ls_o = th.dist_info(torch.from_numpy(theta_tasks), torch.from_numpy(obs.reshape(M, E * H, Do)),
                              (Do, Da, (hidden, hidden)))
    np.testing.assert_allclose(mean.reshape(M, E * H, Da), mu_o.numpy(), rtol=1e-4, atol=2e-5)
    # (2) sampling rule a = mean + eps*exp(log_std) (raw log_std), reported log_std unclipped post-update
    sig = np.exp(theta_tasks[:, -Da:])[:, None, None, :]
    np.testing.assert_allclose(act, mean + noise * sig, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(ph.log_std.cpu().numpy(), theta_tasks[:, -Da:], rtol=0, atol=0)
    # (3) env transitions with the kernel's actions
    if env_name == 'point':
        goals = sampler.vec_env.task_params_per_task.cpu().numpy().astype(np.float64)
        n_bad = 0
        for m in range(M):
            for e in range(E):
                o = nh.NormalizedEnv(nh.PointEnvCorner())
                o.set_task(goals[m])
                for t in range(H):
                    o._wrapped_env._state = obs[m, e, t].astype(np.float64)
                    nxt, r, _, _ = o.step(act[m, e, t].astype(np.float64))
                    if t + 1 < H:
                        np.testing.assert_allclose(obs[m, e, t + 1], nxt, rtol=0, atol=1e-6)
                    n_bad += abs(r - rew[m, e, t]) > 1e-5
        assert n_bad <= 2
    else:
        dirs = sampler.vec_env.task_params_per_task.cpu().numpy()[:, 0]
        info = ph.info.cpu().numpy().reshape(2, M, E, H)
        for t in range(H - 1):
            # rebuild the full state is impossible from obs alone (x is not observed) -> track x separately
            pass
        # full-state replay from the reset state: inject known init states instead
        init = np.zeros((M, E, 18), dtype=np.float32)
        init[..., :9] = rng.uniform(-.1, .1, size=(M, E, 9))
        init[..., 9:] = 0.1 * rng.randn(M, E, 9)
        sampler.inject(noise=noise, init_state=init)
        paths = sampler.obtain_samples()
        ph = paths.phase
        obs = ph.obs.cpu().numpy().reshape(M, E, H, Do)
        act = ph.act.cpu().numpy().reshape(M, E, H, Da)
        rew = ph.rew.cpu().numpy().reshape(M, E, H)
        info = ph.info.cpu().numpy().reshape(2, M, E, H)
        qpos, qvel = init[..., :9].copy(), init[..., 9:].copy()
        np.testing.assert_allclose(obs[:, :, 0], cs.get_obs(qpos, qvel), rtol=0, atol=0)
        for t in range(H):
            u = np.clip(np.float32(-1.0) + (act[:, :, t] + np.float32(10.0)) * np.float32(2.0) / np.float32(20.0), -1, 1)
            qpos, qvel, r, rr, rc = cs.step(qpos, qvel, u.astype(np.float32), dirs[:, None].astype(np.float32))
            np.testing.assert_allclose(rew[:, :, t], r, rtol=1e-3, atol=2e-4)
            np.testing.assert_allclose(info[0, :, :, t], rr, rtol=1e-3, atol=2e-4)
            np.testing.assert_allclose(info[1, :, :, t], rc, rtol=1e-4, atol=1e-6)
            if t + 1 < H:
                np.testing.assert_allclose(obs[:, :, t + 1], cs.get_obs(qpos, qvel), rtol=1e-4, atol=2e-5)
                # re-glue the replay to the kernel state that is observable (everything except x)
                qpos[..., 1:] = obs[:, :, t + 1, :8]
                qvel[...] = obs[:, :, t + 1, 8:]


def test_rollout_philox_statistics():
    """In-kernel Philox noise / reset states: right moments, different per phase, reproducible per seed."""
    torch = _cuda()
    env, policy, sampler, proc = _make_stack('point', 40, 20, 100, reset_mode='device', seed=11)
    sampler.update_tasks()
    p1 = sampler.obtain_samples().phase
    eps = ((p1.act - p1.mean) / torch.exp(p1.log_std).unsqueeze(1)).cpu().numpy().ravel()
    assert abs(eps.mean()) < 0.01 and abs(eps.std() - 1.0) < 0.01
    assert abs(np.mean(eps ** 3)) < 0.05 and abs(np.mean(eps ** 4) - 3.0) < 0.1
    s0 = p1.obs.view(40, 20, 100, 2)[:, :, 0].cpu().numpy()
    assert s0.min() >= -0.2 and s0.max() <= 0.2 and abs(s0.mean()) < 0.02 and abs(s0.std() - 0.4 / math.sqrt(12)) < 0.01
    p2 = sampler.obtain_samples().phase
    assert not torch.equal(p1.act, p2.act)
    env, policy2, sampler2, _ = _make_stack('point', 40, 20, 100, reset_mode='device', seed=11)
    policy2.set_params(policy.get_param_values())
    sampler2.vec_env.set_tasks(sampler.vec_env.tasks)
    q1 = sampler2.obtain_samples().phase
    assert torch.equal(q1.act, p1.act) and torch.equal(q1.obs, p1.obs)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', list('abcde'))
def test_process_samples_matches_reference_golden(golden_dir, case):
    torch = _cuda()
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    g = _load(golden_dir, 'process_samples.npz')
    pre = 'case_%s_' % case
    cfg = {k: g[pre + 'cfg_' + k].item() for k in ('M', 'E', 'H', 'Do', 'Da', 'discount', 'gae_lambda',
                                                    'normalize_adv', 'positive_adv')}
    M, E, H = cfg['M'], cfg['E'], cfg['H']
    paths = OrderedDict()
    for m in range(M):
        paths[m] = [dict(observations=g[pre + 'obs'][m, e], actions=g[pre + 'act'][m, e], rewards=g[pre + 'rew'][m, e],
                         env_infos={}, agent_infos={}) for e in range(E)]
    base = LinearFeatureBaseline()
    proc = MetaSampleProcessor(base, cfg['discount'], cfg['gae_lambda'], bool(cfg['normalize_adv']),
                               bool(cfg['positive_adv']))
    data = proc.process_samples(paths, log=False)
    assert len(data) == M and len(data[0].keys()) == 8
    ret = np.stack([d['returns'] for d in data])
    adv = np.stack([d['advantages'] for d in data])
    np.testing.assert_allclose(ret, g[pre + 'returns'], rtol=2e-7, atol=1e-6)            # float32 rounding of f64 scan
    coeffs = data[0].phase.coeffs.cpu().numpy()
    pred_scale = np.abs(g[pre + 'returns']).max()
    np.testing.assert_allclose(adv, g[pre + 'advantages'], rtol=1e-4, atol=1e-4 * max(1.0, np.abs(g[pre + 'advantages']).max()) * 0.1)
    assert rel_err(adv, g[pre + 'advantages']) < 1e-5
    assert rel_err(coeffs, g[pre + 'coeffs']) < 1e-4, rel_err(coeffs, g[pre + 'coeffs'])
    np.testing.assert_allclose(np.stack([d['adj_avg_rewards'] for d in data]), g[pre + 'adj_avg_rewards'], rtol=1e-5, atol=1e-6)
    np.testing.assert_array_equal(np.stack([d['observations'] for d in data]).reshape(M, E, H, -1), g[pre + 'obs'])
    np.testing.assert_allclose(np.asarray(base.get_param_values()), g[pre + 'coeffs'][-1], rtol=1e-3, atol=1e-6)


def test_process_samples_properties_full_size():
    """BASELINE.json configs[1] size (40x20x100): size-independent properties."""
    torch = _cuda()
    from promp_b200.samplers.device_data import PhaseData
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    M, E, H, Do = 40, 20, 100, 2
    gen = torch.Generator(device='cuda').manual_seed(0)
    ph = PhaseData(M, E, H, Do, 2, torch.device('cuda'))
    ph.obs.copy_(torch.randn(M, E * H, Do, generator=gen, device='cuda'))
    ph.rew.copy_(torch.randn(M, E * H, generator=gen, device='cuda'))
    # gamma = lambda = 1, zero baseline: adv[t] = sum_{k>=t} r[k] (ref tests/test_samplers.py:326-342)
    run_process_kernel(ph, 1.0, 1.0, 1e-5, 0, False, False)
    r = ph.rew.view(M, E, H).double()
    want = torch.flip(torch.cumsum(torch.flip(r, [2]), 2), [2])
    assert torch.allclose(ph.adv.view(M, E, H).double(), want, atol=1e-4)
    assert torch.allclose(ph.returns.view(M, E, H).double(), want, atol=1e-4)
    # normalised advantages: zero mean, unit (population) std per task
    run_process_kernel(ph, 0.99, 0.97, 1e-5, 1, True, False)
    a = ph.adv.double()
    assert a.mean(1).abs().max() < 1e-5 and (a.std(1, unbiased=False) - 1).abs().max() < 1e-4
    # linearity of returns in the rewards
    ret1 = ph.returns.clone()
    ph.rew.mul_(3.0)
    run_process_kernel(ph, 0.99, 0.97, 1e-5, 1, True, False)
    assert torch.allclose(ph.returns, 3.0 * ret1, rtol=1e-5, atol=1e-5)
    # advantages are invariant to reward scaling after normalisation (baseline fit is linear in the target)
    assert torch.allclose(ph.adv.double(), a, atol=2e-4)
    # positive shift
    run_process_kernel(ph, 0.99, 0.97, 1e-5, 1, True, True)
    assert abs(float(ph.adv.min()) - 1e-8) < 1e-6
    # stats: undiscounted return sums agree with torch
    st = ph.stats.cpu().numpy()
    G = ph.rew.view(M, E, H).double().sum(2)
    np.testing.assert_allclose(st[:, 1], G.sum(1).cpu().numpy(), rtol=1e-9, atol=1e-6)
    np.testing.assert_allclose(st[:, 3], G.max(1).values.cpu().numpy(), rtol=1e-9, atol=1e-6)


# ------------------------------------------------------------------------------------------------
def _random_phase(torch, M, N, Do, Da, theta, seed, hidden=64, perturb=1.0):
    """Synthetic sampling-phase data whose old distribution is close to (perturb=1) or exactly (perturb=0)
    the policy given by theta ([P] shared or [M,P] per task)."""
    from promp_b200.samplers.device_data import PhaseData
    from oracle import tf_half as th
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(M, N, Do, generator=g)
    th_t = torch.as_tensor(theta)
    th_t = th_t.view(1, -1).expand(M, -1) if th_t.dim() == 1 else th_t
    mean, ls = th.dist_info(th_t, obs, (Do, Da, (hidden, hidden)))
    old_mean = mean + perturb * 0.1 * torch.randn(M, N, Da, generator=g)
    old_ls = (ls + perturb * 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
    act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
    adv = torch.randn(M, N, generator=g)
    cpu = dict(obs=obs, act=act, adv=adv, mean=old_mean, log_std=old_ls)
    ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
    ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0])
    ph.adv = adv.cuda()
    return cpu, ph


def _algo(torch, kind, M, Do, Da, hidden=64, S1=1, **kw):
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.meta_algos import ProMP, TRPOMAML
    np.random.seed(1)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(hidden, hidden))
    # make log_std and biases non-trivial
    th0 = policy.theta.cpu().numpy()
    th0 += 0.1 * np.random.RandomState(9).randn(th0.size).astype(np.float32)
    policy.set_params(th0)
    if kind == 'promp':
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, learning_rate=1e-3,
                     num_ppo_steps=5, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False, **kw)
    else:
        algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, step_size=0.01, **kw)
    return policy, algo


@pytest.mark.parametrize('Do,Da,hidden,N', [(2, 2, 64, 333), (17, 6, 64, 200), (2, 2, 32, 130), (17, 6, 32, 97)])
@pytest.mark.parametrize('inner', ['likelihood_ratio', 'log_likelihood'])
def test_adapt_matches_oracle(Do, Da, hidden, N, inner):
    """MAMLAlgo._adapt: theta_i' = theta_i - alpha*grad surr_i, pre-update (shared theta) then post-update
    (per-task theta) - against torch autograd on the CPU (float32)."""
    torch = _cuda()
    from oracle import tf_half as th
    M = 5
    policy, algo = _algo(torch, 'trpo', M, Do, Da, hidden, inner_type=inner)
    dims = (Do, Da, (hidden, hidden))
    cpu, ph = _random_phase(torch, M, N, Do, Da, policy.theta.cpu().numpy(), 1, hidden)
    from promp_b200.samplers.device_data import SamplesData
    samples = [SamplesData(ph, m) for m in range(M)]
    policy.switch_to_pre_update()
    algo._adapt(samples)
    want = th.adapt(policy.theta.cpu().view(1, -1).expand(M, -1).contiguous(), cpu, dims, 0.1, inner)
    got = policy.theta_tasks.cpu()
    g_want = (policy.theta.cpu().view(1, -1) - want) / 0.1
    assert rel_err(algo.last_inner_grad.cpu().numpy(), g_want.numpy()) < 2e-5
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-5, atol=1e-6)
    # second inner step from per-task parameters
    algo._adapt(samples)
    want2 = th.adapt(want, cpu, dims, 0.1, inner)
    np.testing.assert_allclose(policy.theta_tasks.cpu().numpy(), want2.numpy(), rtol=1e-5, atol=2e-6)


def test_likelihood_ratio_is_one_at_first_inner_step():
    """ref tests/test_integration.py:150-175: with pi_old = pi_new the likelihood ratio is 1."""
    torch = _cuda()
    env, policy, sampler, proc = _make_stack('point', 10, 2, 50)
    from promp_b200.meta_algos import ProMP
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=10, num_inner_grad_steps=1)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    paths = sampler.obtain_samples()
    samples = proc.process_samples(paths)
    ph = samples[0].phase
    st = torch.zeros(10, 4, device='cuda')
    algo._grad(ph, policy.theta, 0, 0, stats=st)
    assert torch.allclose(st[:, 2], torch.ones(10, device='cuda'), atol=1e-5)     # mean ratio per task
    assert st[:, 1].abs().max() < 1e-6                                              # KL(old||new) = 0


@pytest.mark.parametrize('Do,Da,hidden,N,S1', [(2, 2, 64, 256, 1), (17, 6, 64, 150, 1), (2, 2, 64, 100, 2),
                                               (17, 6, 32, 90, 1), (2, 2, 32, 70, 2), (4, 2, 64, 300, 1), (4, 2, 32, 130, 1)])
@pytest.mark.parametrize('kind', ['promp', 'trpo'])
def test_meta_gradient_matches_oracle(Do, Da, hidden, N, S1, kind):
    """Second-order meta-gradient (forward chain + exact HVP backward chain) vs torch double-backward.
    The oracle is evaluated in float64 on the same float32 inputs; bar: 1e-4 relative on the gradient."""
    torch = _cuda()
    from oracle import tf_half as th
    M = 4
    policy, algo = _algo(torch, kind, M, Do, Da, hidden, S1=S1)
    dims = (Do, Da, (hidden, hidden))
    theta = policy.theta.cpu().numpy()
    cpus, phases = [], []
    for s in range(S1 + 1):
        c, p = _random_phase(torch, M, N, Do, Da, theta, 10 + s, hidden)
        cpus.append({k: v.double() for k, v in c.items()})
        phases.append(p)
    t64 = torch.tensor(theta, dtype=torch.float64, requires_grad=True)
    coeff = list(algo.inner_kl_coeff) if kind == 'promp' else None
    obj, ikl, okl = th.meta_objective(t64, cpus, dims, 0.1, kind, 0.3, coeff)
    (g_want,) = torch.autograd.grad(obj, t64)
    if kind == 'promp':
        res = algo._objective_pass(phases, want_grad=True)
        terms = algo.loss_terms(res).cpu().numpy()
        assert abs(terms[0] - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
        np.testing.assert_allclose(terms[1:1 + S1], ikl.detach().numpy(), rtol=1e-3, atol=1e-6)
        np.testing.assert_allclose(terms[1 + S1], float(okl), rtol=1e-3, atol=1e-6)
        g_got = res['grad'].cpu().numpy()
    else:
        g_got = algo.eval_gradient(policy.theta, phases, 'loss')
        loss, klv = algo.eval_scalars(policy.theta, phases)
        assert abs(loss - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
        assert abs(klv - float(okl)) < 1e-3 * max(1e-3, abs(float(okl)))
        # constraint gradient too
        (gk_want,) = torch.autograd.grad(th.meta_objective(t64, cpus, dims, 0.1, kind)[2], t64)
        gk_got = algo.eval_gradient(policy.theta, phases, 'kl')
        assert rel_err(gk_got, gk_want.numpy()) < 1e-4, rel_err(gk_got, gk_want.numpy())
    err = rel_err(g_got, g_want.numpy())
    assert err < 1e-4, err
    assert abs(np.linalg.norm(g_got) / np.linalg.norm(g_want.numpy()) - 1) < 1e-4     # grad-norm bar of the north star


def test_adam_tf1_matches_oracle():
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.optimizers import MAMLPPOOptimizer

    class P(object):
        pass
    p = P()
    p.num_params, p.device = 1000, torch.device('cuda')
    g = torch.Generator().manual_seed(0)
    theta0 = torch.randn(1000, generator=g)
    p.theta = theta0.clone().cuda()
    opt = MAMLPPOOptimizer(learning_rate=1e-3)
    opt.build(p)
    adam = th.TF1Adam(1000)
    cur = theta0.clone()
    for i in range(7):
        grad = torch.randn(1000, generator=g) * (10.0 ** (i % 3 - 1))
        opt.apply_gradient(grad.cuda())
        cur = adam.step(cur, grad)
    np.testing.assert_allclose(p.theta.cpu().numpy(), cur.numpy(), rtol=1e-5, atol=1e-7)
    assert int(opt.step.item()) == 7


@pytest.mark.parametrize('Do,Da', [(2, 2), (17, 6)])
def test_promp_optimize_policy_matches_oracle(Do, Da):
    """ProMP.optimize_policy: 5 Adam epochs + stats pass vs the float32 torch restatement."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.samplers.device_data import SamplesData
    M, N = 6, 300
    policy, algo = _algo(torch, 'promp', M, Do, Da)
    dims = (Do, Da, (64, 64))
    theta0 = policy.theta.cpu().clone()
    cpus, all_samples = [], []
    for s in range(2):
        c, p = _random_phase(torch, M, N, Do, Da, theta0.numpy(), 20 + s)
        cpus.append(c)
        all_samples.append([SamplesData(p, m) for m in range(M)])
    adam = th.TF1Adam(theta0.numel())
    want, st = th.promp_optimize(theta0.clone(), cpus, dims, adam, 0.1, 0.3, list(algo.inner_kl_coeff), 5)
    algo.optimize_policy(all_samples, log=False)
    got = policy.theta.cpu()
    # Adam normalises the step: compare the *update*, which is O(lr) per coordinate
    assert rel_err((got - theta0).numpy(), (want - theta0).numpy()) < 2e-3
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=0, atol=2e-5)
    ls = algo.last_stats
    assert abs(ls['loss_before'] - st['loss_before']) < 1e-4 * max(1, abs(st['loss_before']))
    assert abs(ls['loss_after'] - st['loss_after']) < 1e-4 * max(1, abs(st['loss_after']))
    np.testing.assert_allclose(ls['inner_kls'], st['inner_kls'], rtol=2e-3, atol=1e-6)
    assert abs(ls['outer_kl'] - st['outer_kl']) < 2e-3 * max(1e-3, abs(st['outer_kl']))


def test_trpo_maml_optimize_policy_runs_and_matches_first_quantities():
    """TRPO-MAML: loss gradient and one finite-difference Hx against the oracle (the CG result itself is
    dominated by fp32 finite-difference noise, SURVEY.md section 7), then a full optimize_policy."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.samplers.device_data import SamplesData
    M, N, Do, Da = 4, 400, 2, 2
    policy, algo = _algo(torch, 'trpo', M, Do, Da, inner_type='log_likelihood')
    dims = (Do, Da, (64, 64))
    theta0 = policy.theta.cpu().numpy().copy()
    cpus, phases, all_samples = [], [], []
    # like real sampling: phase 0 is drawn from pi_theta, phase 1 from the adapted pi_theta_i'
    c, p = _random_phase(torch, M, N, Do, Da, theta0, 30, perturb=0.0)
    cpus.append(c); phases.append(p)
    adapted = th.adapt(torch.from_numpy(theta0).view(1, -1).expand(M, -1).contiguous(), c, dims, 0.1, 'log_likelihood')
    c, p = _random_phase(torch, M, N, Do, Da, adapted.numpy(), 31, perturb=0.0)
    cpus.append(c); phases.append(p)
    all_samples = [[SamplesData(ph, m) for m in range(M)] for ph in phases]
    orc = th.TRPOMAMLOracle(dims, 0.1, 0.01, 'log_likelihood')
    g_o = orc.gradient(theta0, cpus)
    g_d = algo.eval_gradient(policy.theta, phases, 'loss')
    assert rel_err(g_d, g_o) < 1e-4
    x = g_o / np.linalg.norm(g_o)
    hx_o = orc.Hx(theta0, cpus, x.astype(np.float32))
    hx_d = algo.optimizer.Hx(theta0, phases, x.astype(np.float32))
    assert rel_err(hx_d, hx_o) < 0.2            # both are fp32 central differences with eps = 1e-5
    algo.optimize_policy(all_samples, log=False)
    ls = algo.last_stats
    assert ls['kl_before'] < 1e-6
    assert np.isfinite(ls['loss_after']) and ls['kl'] <= 0.01 + 1e-6
    assert ls['loss_after'] < ls['loss_before'] and not algo.optimizer.last['rejected']
    assert algo.optimizer.last['backtracks'] >= 0
    # same decision sequence as the oracle's host loop
    th_o, st_o = orc.optimize(theta0, cpus)
    assert st_o['rejected'] is False
    assert abs(st_o['loss'] - ls['loss_after']) < 0.05 * abs(ls['loss_before'] - ls['loss_after']) + 1e-5


def test_first_epoch_inner_pass_reuses_adapt_launch_exactly():
    """The inner pass of the first Adam epoch repeats MAMLAlgo._adapt; it skips itself on the device (promp_policy_grad_ex) iff
    the parameters are bit-identical to the ones _adapt used and the step-0 log_std clip is inactive.  Checked: identical
    results with and without the shortcut; a parameter change after _adapt, or an active clip, makes the kernel run (results
    equal the uncached evaluation, not the stale cache)."""
    torch = _cuda()
    from promp_b200.meta_algos import ProMP
    M, E, H = 4, 5, 40

    def evaluate(mutate=None, use_cache=True, ls=None):
        env, policy, sampler, proc = _make_stack('point', M, E, H, seed=11)
        if ls is not None:
            th = policy.theta.clone()
            th[-2:] = ls
            policy.theta.copy_(th)
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                     clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
        np.random.seed(4)
        sampler.update_tasks()
        policy.switch_to_pre_update()
        phases = []
        for step in range(2):
            paths = sampler.obtain_samples()
            samples = proc.process_samples(paths)
            phases.append(samples[0].phase)
            if step == 0:
                algo._adapt(samples)
        assert algo._adapt_cache is not None
        if mutate is not None:
            mutate(policy)
        if not use_cache:
            algo._adapt_cache = None
        res = algo._objective_pass(phases, want_grad=True)
        terms = algo.loss_terms(res).cpu().numpy()
        return res['grad'].cpu().numpy(), terms, algo

    g_c, t_c, algo = evaluate()
    assert algo._adapt_cache is None                      # consumed by the first pass
    g_n, t_n, _ = evaluate(use_cache=False)
    assert np.array_equal(g_c, g_n) and np.array_equal(t_c, t_n)
    bump = lambda pol: pol.theta.add_(1e-3)
    g_c, t_c, _ = evaluate(mutate=bump)
    g_n, t_n, _ = evaluate(mutate=bump, use_cache=False)
    assert np.array_equal(g_c, g_n) and np.array_equal(t_c, t_n)
    g_c, t_c, _ = evaluate(ls=-15.0)                      # below log(1e-6): the step-0 graph clips, _adapt does not
    g_n, t_n, _ = evaluate(ls=-15.0, use_cache=False)
    assert np.array_equal(g_c, g_n) and np.array_equal(t_c, t_n)


def test_fused_meta_update_single_gpu():
    """promp_meta_update (task mean + TF1 Adam in one launch, world = 1) == promp_reduce_tasks + promp_adam_tf1."""
    torch = _cuda()
    from promp_b200 import _lib
    g = torch.Generator(device='cuda').manual_seed(3)
    M, P = 9, 5708
    v = torch.randn(M, P, generator=g, device='cuda')
    theta_a = torch.randn(P, generator=g, device='cuda')
    theta_b = theta_a.clone()
    ma, va, mb, vb = (torch.zeros(P, device='cuda') for _ in range(4))
    sa, sb = (torch.zeros(1, dtype=torch.int32, device='cuda') for _ in range(2))
    ticket = torch.zeros(1, dtype=torch.int32, device='cuda')
    ga, gb = torch.empty(P, device='cuda'), torch.empty(P, device='cuda')
    for it in range(4):
        v.mul_(0.7).add_(0.1)
        _lib.call('promp_meta_update', M, P, _lib.ptr(v), 1.0 / M, _lib.ptr(ga), _lib.ptr(theta_a), _lib.ptr(ma), _lib.ptr(va),
                  _lib.ptr(sa), 1e-3, 0.9, 0.999, 1e-8, 1, 0, 0, None, None, None, _lib.ptr(ticket), _lib.stream())
        _lib.call('promp_reduce_tasks', M, P, _lib.ptr(v), 1.0 / M, _lib.ptr(gb), _lib.stream())
        _lib.call('promp_adam_tf1', P, _lib.ptr(theta_b), _lib.ptr(gb), _lib.ptr(mb), _lib.ptr(vb), _lib.ptr(sb), 1e-3, 0.9, 0.999,
                  1e-8, _lib.stream())
        assert torch.equal(ga, gb) and torch.equal(theta_a, theta_b) and torch.equal(ma, mb) and torch.equal(va, vb)
    assert int(sa.item()) == 4 and int(ticket.item()) == 0


def test_device_cg_and_line_search_kernels(golden_dir):
    """promp_cg_init / promp_cg_step against the UNMODIFIED reference's conjugate_gradients outputs
    (tests/golden/tf_half_known.npz: cg_x10, cg_x3, early exit at residual_tol), driven with grad_plus = A p, grad_minus = 0,
    two_eps = 1 (so that Hx(p) = A p); then promp_trpo_step and the accept / violate / restore rule of promp_trpo_select
    (conjugate_gradient_optimizer.py:262-300) on hand-made candidate tables."""
    torch = _cuda()
    from promp_b200 import _lib
    g = _load(golden_dir, 'tf_half_known.npz')
    A = torch.from_numpy(g['cg_A']).cuda()
    b = torch.from_numpy(g['cg_b']).cuda()
    n = b.numel()
    zero = torch.zeros(n, device='cuda')

    def cg(iters, tol):
        p, r, x = (torch.empty(n, device='cuda') for _ in range(3))
        scal = torch.zeros(4, device='cuda')
        _lib.call('promp_cg_init', n, _lib.ptr(b), _lib.ptr(p), _lib.ptr(r), _lib.ptr(x), _lib.ptr(scal), _lib.stream())
        for _ in range(iters):
            z = (A @ p).contiguous()
            _lib.call('promp_cg_step', n, _lib.ptr(z), _lib.ptr(zero), 1.0, 0.0, _lib.ptr(p), _lib.ptr(r), _lib.ptr(x),
                      _lib.ptr(scal), float(tol), _lib.stream())
        return x.cpu().numpy(), scal.cpu().numpy()
    for iters, key, tol in ((10, 'cg_x10', 1e-10), (3, 'cg_x3', 1e-10), (200, 'cg_x_tol', 1e-6)):
        x, scal = cg(iters, tol)
        assert rel_err(x, g[key]) < 2e-5, (key, rel_err(x, g[key]))       # float32 vectors, float64-accumulated dots
        assert (scal[1] == 1.0) == (key == 'cg_x_tol')                       # the early exit fired only with the loose tolerance
    # step length: beta = sqrt(2 delta / (x.Hx + 1e-8))
    x = torch.from_numpy(g['cg_x10']).cuda()
    hx = (A @ x).contiguous()
    step, scal = torch.empty(n, device='cuda'), torch.zeros(4, device='cuda')
    _lib.call('promp_trpo_step', n, _lib.ptr(hx), _lib.ptr(zero), 1.0, 0.0, _lib.ptr(x), 0.01, _lib.ptr(step), _lib.ptr(scal), _lib.stream())
    beta = np.sqrt(2.0 * 0.01 / (float(g['cg_x10'].dot(g['cg_A'].dot(g['cg_x10']))) + 1e-8))
    np.testing.assert_allclose(step.cpu().numpy(), beta * g['cg_x10'], rtol=2e-6)
    assert scal[3].item() == 0.0
    _lib.call('promp_trpo_step', n, _lib.ptr(-hx), _lib.ptr(zero), 1.0, 0.0, _lib.ptr(x), 0.01, _lib.ptr(step), _lib.ptr(scal), _lib.stream())
    assert scal[3].item() == 1.0                      # x.Hx < 0 -> NaN step -> the verdict kernel rejects
    # line-search verdicts: rows are [loss, (inner kl), kl]; loss_before = 1.0, delta = 0.01
    prev = torch.arange(n, dtype=torch.float32, device='cuda')
    cands = torch.stack([prev + 10 * (k + 1) for k in range(4)]).contiguous()
    base = torch.tensor([1.0, 0.0, 0.001], device='cuda')

    def verdict(rows, k0=0, nan_beta=False, kmax=15):
        terms = torch.tensor(rows, dtype=torch.float32, device='cuda')
        sc = torch.tensor([0, 0, 0.5, 1.0 if nan_beta else 0.0], dtype=torch.float32, device='cuda')
        out = torch.full((n,), -7.0, device='cuda')
        res = torch.zeros(8, device='cuda')
        _lib.call('promp_trpo_select', n, len(rows), 3, k0, kmax, _lib.ptr(terms), _lib.ptr(base), 0.01, _lib.ptr(prev),
                  _lib.ptr(cands), _lib.ptr(sc), _lib.ptr(out), _lib.ptr(res), _lib.stream())
        return out.cpu().numpy(), res.cpu().numpy()
    ok, bad_loss, bad_kl = [0.9, 0, 0.005], [1.1, 0, 0.005], [0.9, 0, 0.02]
    out, res = verdict([ok, ok, ok, ok])
    assert res[4] == 0 and res[5] == 0 and res[6] == 0 and np.array_equal(out, cands[0].cpu().numpy()) and res[2] == np.float32(0.9)
    out, res = verdict([bad_loss, bad_kl, ok, ok])
    assert res[4] == 2 and res[5] == 0 and np.array_equal(out, cands[2].cpu().numpy())
    out, res = verdict([bad_loss, bad_kl, bad_kl, bad_loss])
    assert res[4] == -1 and res[6] == 1 and np.all(out == -7.0)                       # undecided: parameters untouched
    out, res = verdict([bad_loss, bad_kl, ok], k0=12)                                  # third group accepts k = 14
    assert res[4] == 14 and np.array_equal(out, cands[2].cpu().numpy())
    out, res = verdict([bad_loss, bad_kl, bad_kl], k0=12)                              # budget exhausted -> restored
    assert res[5] == 1 and res[6] == 0 and np.array_equal(out, prev.cpu().numpy()) and res[2] == 1.0
    out, res = verdict([[0.9, 0, 0.01]])                                               # kl == delta: accepted by the loop, then "violated"
    assert res[4] == 0 and res[5] == 1 and np.array_equal(out, prev.cpu().numpy())
    out, res = verdict([[float('nan'), 0, 0.001], ok])                                 # NaN loss is never accepted
    assert res[4] == 1
    out, res = verdict([ok, ok], nan_beta=True)
    assert res[5] == 1 and res[4] == -1 and np.array_equal(out, prev.cpu().numpy())


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('env_name', ['point', 'cheetah'])
def test_trainer_end_to_end(env_name):
    """Full meta-iterations through the reference-shaped classes; reference logging keys present."""
    torch = _cuda()
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    logger.set_quiet(True)
    M, E, H = 5, 4, 100
    env, policy, sampler, proc = _make_stack(env_name, M, E, H)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                 num_ppo_steps=5, clip_eps=0.3, target_inner_step=0.01, init_inner_kl_penalty=5e-4,
                 adaptive_inner_kl_penalty=False)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                      num_inner_grad_steps=1)
    theta0 = policy.theta.clone()
    trainer.train()
    kv = logger.last_dump()
    for key in ('Step_0-AverageReturn', 'Step_1-AverageReturn', 'Step_0-AveragePolicyStd', 'LossBefore', 'LossAfter',
                'KLInner', 'KLCoeffInner', 'Time-Sampling', 'Time-OuterStep', 'ItrTime', 'n_timesteps'):
        assert key in kv, key
    assert kv['n_timesteps'] == 3 * 2 * M * E * H
    assert torch.isfinite(policy.theta).all() and not torch.equal(policy.theta, theta0)
    assert np.isfinite(kv['LossAfter'])
    # policy pickles through get/set state (policies/base.py:205-215)
    import pickle
    pol2 = pickle.loads(pickle.dumps(policy))
    assert torch.equal(pol2.theta, policy.theta)


@pytest.mark.parametrize('env_name', ['point', 'cheetah'])
def test_trainer_cuda_graph_mode(env_name):
    """Trainer(use_cuda_graph=True): the device part of the iteration replayed as one CUDA graph, host inputs drawn
    from numpy in the reference's order, logged scalars read back in one copy - same keys, consistent values."""
    torch = _cuda()
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    logger.set_quiet(True)
    M, E, H = 6, 5, 40
    env, policy, sampler, proc = _make_stack(env_name, M, E, H)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                 num_ppo_steps=5, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=1,
                      num_inner_grad_steps=1, use_cuda_graph=True)
    step = trainer.capture_graph(warmup=2, log=True)
    np.random.seed(123)
    theta0 = policy.theta.clone()
    obs_prev = None
    for itr in range(3):
        phases = step(itr)
        kv = dict(logger.getkvs())
        for key in ('Step_0-AverageReturn', 'Step_1-AverageReturn', 'Step_0-StdReturn', 'Step_1-MaxReturn',
                    'Step_0-AveragePolicyStd', 'LossBefore', 'LossAfter', 'KLInner', 'KLCoeffInner', 'n_timesteps'):
            assert key in kv and np.isfinite(kv[key]), key
        # logged values agree with the device buffers they summarise
        for s, ph in enumerate(phases):
            ret = ph.rew.view(M * E, H).double().sum(1)
            assert abs(kv['Step_%d-AverageReturn' % s] - float(ret.mean())) < 1e-4 * max(1.0, abs(float(ret.mean())))
            assert abs(kv['Step_%d-MaxReturn' % s] - float(ret.max())) < 1e-4 * max(1.0, abs(float(ret.max())))
            assert kv['Step_%d-NumTrajs' % s] == M * E
        if env_name == 'cheetah':
            assert 'Step_0-AvgForwardVel' in kv and 'Step_1-AvgCtrlCost' in kv
        # fresh noise / reset states on every replay
        cur = phases[0].obs.clone()
        if obs_prev is not None:
            assert not torch.equal(cur, obs_prev)
        obs_prev = cur
    assert not torch.equal(policy.theta, theta0) and torch.isfinite(policy.theta).all()
    # numpy stream consumption == reference order: tasks, then per phase (M*E resets + M*E discarded resets)
    probe = np.random.uniform(size=3)
    np.random.seed(123)
    inner = env._wrapped_env
    for itr in range(3):
        env.sample_tasks(M)
        for s in range(2):
            inner.host_reset_states(M * E)
            inner.host_reset_states(M * E)
    assert np.array_equal(probe, np.random.uniform(size=3))
    # reset states of the last replay are exactly the host draws
    np.random.seed(7)
    phases = step(3)
    np.random.seed(7)
    env.sample_tasks(M)
    want = inner.host_reset_states(M * E).astype(np.float32)
    got = phases[0].obs.view(M * E, H, -1)[:, 0].cpu().numpy()
    if env_name == 'point':
        np.testing.assert_array_equal(got, want)
    else:
        np.testing.assert_array_equal(got, np.concatenate([want[:, 1:9], want[:, 9:]], axis=1))


def test_hidden16_runs_zero_padded_and_matches_oracle():
    """hidden_sizes=(16,16) (the reference's test configuration, tests/test_integration.py:88) runs on the 32-wide
    kernels zero-padded: padded parameters stay exactly zero, logical ones match the (16,16) oracle."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.meta_algos import ProMP
    from promp_b200.samplers.device_data import PhaseData, SamplesData
    M, N, Do, Da = 4, 150, 2, 2
    np.random.seed(2)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(16, 16))
    assert policy.hidden == 32 and policy.num_params_logical == th.num_params(Do, Da, (16, 16))
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                 num_ppo_steps=3, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    dims = (Do, Da, (16, 16))
    theta_l = policy.unpad_flat(policy.theta.cpu().numpy()).copy()
    vals = policy.get_param_values()
    assert vals['mean_network/hidden_1/kernel'].shape == (16, 16)
    cpus, phases = [], []
    for s in range(2):
        g = torch.Generator().manual_seed(50 + s)
        obs = torch.randn(M, N, Do, generator=g)
        mean, ls = th.dist_info(torch.from_numpy(theta_l).view(1, -1).expand(M, -1), obs, dims)
        old_mean = mean + 0.1 * torch.randn(M, N, Da, generator=g)
        old_ls = (ls + 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
        act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
        adv = torch.randn(M, N, generator=g)
        cpus.append({k: v.double() for k, v in dict(obs=obs, act=act, adv=adv, mean=old_mean, log_std=old_ls).items()})
        ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
        ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0]); ph.adv = adv.cuda()
        phases.append(ph)
    t64 = torch.tensor(theta_l, dtype=torch.float64, requires_grad=True)
    obj, _, _ = th.meta_objective(t64, cpus, dims, 0.1, 'promp', 0.3, list(algo.inner_kl_coeff))
    (g_want,) = torch.autograd.grad(obj, t64)
    res = algo._objective_pass(phases, want_grad=True)
    g_pad = res['grad'].cpu().numpy()
    assert rel_err(policy.unpad_flat(g_pad), g_want.numpy()) < 1e-4
    mask = np.ones(policy.num_params, dtype=bool)
    mask[policy._pad_index_np] = False
    assert np.all(g_pad[mask] == 0.0)
    algo.optimize_policy([[SamplesData(p, m) for m in range(M)] for p in phases], log=False)
    assert np.all(policy.theta.cpu().numpy()[mask] == 0.0)           # padding is preserved by Adam
    # round trip through the reference-style accessors
    policy.set_params(policy.get_param_values())
    assert np.all(policy.theta.cpu().numpy()[mask] == 0.0)


def test_raw_env_without_normalize_wrapper(golden_dir):
    """The reference's tests use un-wrapped envs: the env kernels take normalize_actions = 0 and then apply only
    the env's own clip.  MetaPointEnv: s' = s + clip(a, +-0.1), r = -|s'|, done near the origin."""
    torch = _cuda()
    from promp_b200.envs import MetaPointEnv
    from promp_b200.samplers import MetaDeviceEnvExecutor
    np.random.seed(0)
    n = 16
    ex = MetaDeviceEnvExecutor(MetaPointEnv(), n, 1, max_path_length=10 ** 6)
    ex.set_tasks([{}] * n)
    obs0 = np.asarray(ex.reset())
    assert np.abs(obs0).max() <= 2.0
    act = np.random.uniform(-0.3, 0.3, size=(n, 2))
    obs, rew, dones, _ = ex.step(act)
    want = obs0.astype(np.float32) + np.clip(act, -0.1, 0.1).astype(np.float32)
    np.testing.assert_allclose(np.asarray(obs), want, atol=1e-6)
    np.testing.assert_allclose(np.asarray(rew), -np.sqrt((want ** 2).sum(1)), rtol=1e-5)


def test_p2p_allreduce_two_gpus():
    """promp_allreduce_p2p (NVLink peer memory, rank-ordered, graph-capturable) vs NCCL on 2 GPUs; skipped on a
    single-GPU box."""
    torch = _cuda()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', '29547', os.path.join(root, 'tests', '_p2p_worker.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=200)
    assert r.returncode == 0 and 'rank 0 p2p ok' in r.stdout and 'rank 1 p2p ok' in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


def test_emaml_exploration_term_matches_oracle():
    """TRPOMAML(exploration=True) = E-MAML (ref meta_algos/trpo_maml.py:137-144): objective and gradient incl. the
    initial-log-likelihood term weighted by the last phase's mean adjusted reward."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    M, N, Do, Da = 4, 200, 2, 2
    policy, algo = _algo(torch, 'trpo', M, Do, Da, exploration=True)
    dims = (Do, Da, (64, 64))
    theta = policy.theta.cpu().numpy()
    cpus, phases = [], []
    for s in range(2):
        c, p = _random_phase(torch, M, N, Do, Da, theta, 70 + s)
        # rewards -> the processing kernel's per-task sums feed adj_avg_rewards
        g = torch.Generator().manual_seed(90 + s)
        rew = torch.randn(M, N, generator=g) + torch.arange(M).view(-1, 1).float()
        p.rew.copy_(rew)
        adv_keep = p.adv.clone()
        run_process_kernel(p, 0.99, 1.0, 1e-5, 1, True, False)
        p.adv = adv_keep
        r64 = rew.double()
        c = {k: v.double() for k, v in c.items()}
        c['adj_avg_rewards'] = (r64 - r64.mean()) / (r64.std(unbiased=False) + 1e-8)
        cpus.append(c); phases.append(p)
    t64 = torch.tensor(theta, dtype=torch.float64, requires_grad=True)
    obj, _, okl = th.meta_objective(t64, cpus, dims, 0.1, 'trpo', exploration=True)
    (g_want,) = torch.autograd.grad(obj, t64)
    obj_plain = th.meta_objective(t64, cpus, dims, 0.1, 'trpo')[0]
    assert abs(float(obj) - float(obj_plain)) > 1e-3          # the term is actually exercised
    loss, klv = algo.eval_scalars(policy.theta, phases)
    assert abs(loss - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
    g_got = algo.eval_gradient(policy.theta, phases, 'loss')
    assert rel_err(g_got, g_want.detach().numpy()) < 1e-4


def test_policy_kernels_deterministic_and_batch_independent():
    """(i) Two launches on the same inputs are bitwise identical (fixed-order reductions, no atomics on data);
    (ii) a task's adapted parameters / HVP do not depend on which other tasks share the launch (tile scheduling
    crosses task boundaries inside CTAs): M = 96 tasks vs the same tasks run 6 at a time."""
    torch = _cuda()
    Do, Da, N = 2, 2, 1000
    M = 96
    policy, algo = _algo(torch, 'promp', M, Do, Da)
    theta = policy.theta.cpu().numpy()
    _, ph = _random_phase(torch, M, N, Do, Da, theta, 3)
    P = policy.num_params
    vec = 0.01 * torch.randn(M, P, generator=torch.Generator().manual_seed(1)).cuda()
    outs = []
    for rep in range(2):
        g = torch.empty(M, P, device='cuda'); newp = torch.empty(M, P, device='cuda'); hv = torch.empty(M, P, device='cuda')
        st = torch.zeros(M, 4, device='cuda')
        algo._grad(ph, policy.theta, 0, 0, clip_log_std=1, grad=g, out_params=newp, sgd_lr=0.1, stats=st)
        algo._hvp(ph, newp, P, vec, hv, 5e-4, 0)
        outs.append((g, newp, hv, st))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    # the same tasks in small launches
    from promp_b200.samplers.device_data import PhaseData
    sub = 6
    pol2, algo2 = _algo(torch, 'promp', sub, Do, Da)
    pol2.set_params(policy.get_param_values())
    for m0 in (0, 42, 90):
        p2 = PhaseData(sub, 1, N, Do, Da, torch.device('cuda'))
        sl = slice(m0, m0 + sub)
        p2.obs.copy_(ph.obs[sl]); p2.act.copy_(ph.act[sl]); p2.mean.copy_(ph.mean[sl]); p2.log_std.copy_(ph.log_std[sl])
        p2.adv = ph.adv[sl].contiguous()
        g = torch.empty(sub, P, device='cuda'); newp = torch.empty(sub, P, device='cuda'); hv = torch.empty(sub, P, device='cuda')
        algo2._grad(p2, pol2.theta, 0, 0, clip_log_std=1, grad=g, out_params=newp, sgd_lr=0.1)
        algo2._hvp(p2, newp, P, vec[sl].contiguous(), hv, 5e-4, 0)
        # different tile->CTA assignment changes the summation order of the partials (and of the 3xTF32 terms): equal to
        # fp32 round-off, far inside the 1e-4 parity bar
        assert rel_err(g.cpu().numpy(), outs[0][0][sl].cpu().numpy()) < 5e-6
        assert rel_err(hv.cpu().numpy(), outs[0][2][sl].cpu().numpy()) < 5e-6


def test_processor_argument_contract():
    """process_samples keeps the reference's argument contract (meta_sample_processor.py:25); variable-length paths are
    accepted (see the ragged tests below)."""
    _cuda()
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline, ZeroBaseline
    rng = np.random.RandomState(0)
    paths = {0: [dict(observations=rng.randn(L, 2), actions=rng.randn(L, 2), rewards=rng.randn(L), env_infos={}, agent_infos={})
                 for L in (5, 7)]}
    data = MetaSampleProcessor(LinearFeatureBaseline()).process_samples(paths)
    assert len(data) == 1 and data[0]['advantages'].shape == (12,)
    with pytest.raises(AssertionError):
        MetaSampleProcessor(ZeroBaseline()).process_samples([paths[0]])       # must be a dict (meta_sample_processor.py:25)
    with pytest.raises(ValueError):
        MetaSampleProcessor(ZeroBaseline()).process_samples({0: paths[0], 1: []})   # a task without a completed path


def test_early_terminating_env_end_to_end():
    """MetaPointEnv (done near the origin, point_env_2d.py:49-53) through the stepwise sampler's "collect until
    >= M*E*H samples in completed paths" loop (meta_sampler.py:87-137), the ragged processor, adapt and one ProMP
    optimisation: variable-length paths all the way down, finite results, per-task sample counts as sampled."""
    torch = _cuda()
    from promp_b200.envs import MetaPointEnv, normalize
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.meta_algos import ProMP
    np.random.seed(3)
    M, E, H = 4, 5, 12
    env = normalize(MetaPointEnv())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1.0, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=2)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    all_samples = []
    theta0 = policy.theta.clone()
    for step in range(2):
        paths = sampler.obtain_samples()
        lens = [[len(p['rewards']) for p in paths[m]] for m in range(M)]
        assert sum(map(sum, lens)) >= M * E * H and all(max(l) <= H for l in lens)
        data = proc.process_samples(paths)
        assert [len(d['advantages']) for d in data] == [sum(l) for l in lens]
        assert all(np.isfinite(d['advantages']).all() for d in data)
        all_samples.append(data)
        if step == 0:
            algo._adapt(data)
    algo.optimize_policy(all_samples, log=False)
    th1 = policy.theta
    assert torch.isfinite(th1).all() and not torch.equal(th1, theta0)


@pytest.mark.parametrize('exploration', [False, True])
def _origin_seeking_policy(torch, M):
    """theta with mean ~= -100 * obs through the (near-linear) tanh layers and sigma = e^-10: on normalize(MetaPointEnv)
    (a_env = clip(0.01 a, +-0.1), envs/normalized_env.py:109-114) the point walks 0.1 per step towards the origin and lands
    within 0.01 of it -> early `done` after <= 21 steps."""
    from promp_b200.policies import MetaGaussianMLPPolicy
    from oracle import tf_cases
    np.random.seed(0)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
    par = tf_cases.unflatten(np.zeros(policy.num_params_logical, np.float32), 2, 2, 64)
    c = 0.01
    par['mean_network/hidden_0/kernel'][0, 0] = par['mean_network/hidden_0/kernel'][1, 1] = c
    par['mean_network/hidden_1/kernel'][0, 0] = par['mean_network/hidden_1/kernel'][1, 1] = 1.0
    par['mean_network/output/kernel'][0, 0] = par['mean_network/output/kernel'][1, 1] = -100.0 / c
    par['log_std_network/log_std_var'][:] = -10.0
    policy.set_params(par)
    return policy


def test_fused_early_termination_matches_reference_rule():
    """MetaPointEnv through promp_rollout_early_term + promp_paths_finalize (reset_mode='device'): the device-built path
    table and compacted tensors equal a host re-statement of the reference loop (meta_sampler.py:87-137: step all envs, append a
    path at the step it completes in env order, stop when the completed paths hold >= M*E*H samples, drop unfinished ones)
    applied to the recorded timelines; env dynamics, in-kernel resets, horizon logic checked on the timelines themselves; the
    processing kernel and a ProMP step run on the result."""
    torch = _cuda()
    from promp_b200.envs import normalize, MetaPointEnv
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.samplers.device_data import DeviceRaggedPhaseData
    M, E, H = 3, 6, 25
    policy = _origin_seeking_policy(torch, M)
    env = normalize(MetaPointEnv())
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          reset_mode='device', seed=5)
    assert sampler._fused_early_ok() and not sampler._fused_ok()
    sampler.update_tasks()
    policy.switch_to_pre_update()
    paths = sampler.obtain_samples()
    ph = paths.phase
    assert isinstance(ph, DeviceRaggedPhaseData)
    tl = ph.timeline
    T = 2 * H - 1
    done = tl['done'].cpu().numpy().astype(bool)
    t_obs, t_act, t_rew = tl['obs'].cpu().numpy(), tl['act'].cpu().numpy(), tl['rew'].cpu().numpy()
    # ---- timelines: dynamics, done rule, resets
    for m in range(M):
        for e in range(E):
            ts = 0
            for t in range(T):
                s = t_obs[m, e, t].astype(np.float64)
                a_env = np.clip(0.01 * t_act[m, e, t].astype(np.float64), -0.1, 0.1)    # NormalizedEnv map onto [-0.1, 0.1]
                s2 = s + a_env
                assert abs(t_rew[m, e, t] + np.linalg.norm(s2)) < 1e-5
                ts += 1
                want_done = (abs(s2[0]) < 0.01 and abs(s2[1]) < 0.01) or ts >= H
                assert bool(done[m, e, t]) == want_done, (m, e, t)
                if t + 1 < T:
                    nxt = t_obs[m, e, t + 1]
                    if want_done:
                        assert np.all(np.abs(nxt) <= 2.0) and np.abs(nxt - s2).max() > 1e-3      # fresh U(-2,2)^2 reset state
                        ts = 0
                    else:
                        np.testing.assert_allclose(nxt, s2, atol=2e-6)
    assert done.any() and (done.sum(-1) > 1).any()            # early terminations happened (several paths per slot)
    # ---- host re-statement of the collect-until-enough rule on the same timelines
    from test_paths_finalize import collect_until
    total = M * E * H
    rule = collect_until(done, total)
    assert rule.reached
    want_paths, t_star = rule.paths, rule.t_star
    cut = ph.cut.cpu().numpy()
    assert cut[0] == t_star and cut[1] == 1
    n_paths, n_valid, off = ph.n_paths_host, ph.n_valid_host, ph.path_off_host
    obs_r, act_r, rew_r, done_r = ph.obs.cpu().numpy(), ph.act.cpu().numpy(), ph.rew.cpu().numpy(), ph.done.cpu().numpy()
    for m in range(M):
        assert n_paths[m] == len(want_paths[m]) and n_valid[m] == sum(p[2] for p in want_paths[m])
        pos = 0
        for k, (e, s0, L) in enumerate(want_paths[m]):
            assert off[m, k] == pos and off[m, k + 1] == pos + L
            np.testing.assert_array_equal(obs_r[m, pos:pos + L], t_obs[m, e, s0:s0 + L])
            np.testing.assert_array_equal(act_r[m, pos:pos + L], t_act[m, e, s0:s0 + L])
            np.testing.assert_array_equal(rew_r[m, pos:pos + L], t_rew[m, e, s0:s0 + L])
            assert done_r[m, pos + L - 1] == 1 and done_r[m, pos:pos + L - 1].sum() == 0
            pos += L
        # the lazy per-task path list the reference-shaped callers see
        assert len(paths[m]) == len(want_paths[m])
        np.testing.assert_array_equal(paths[m][0]['observations'], t_obs[m, want_paths[m][0][0], :want_paths[m][0][2]])
    assert int(n_valid.sum()) >= total and int(n_valid.sum()) - total < M * E * H      # enough, not everything
    # ---- downstream kernels take the device-built ragged phase
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    samples = proc.process_samples(paths, log='all', log_prefix='x-')
    adv = ph.adv.cpu().numpy()
    for m in range(M):
        a = adv[m, :n_valid[m]]
        assert np.isfinite(a).all() and abs(a.mean()) < 1e-4 and abs(a.std() - 1) < 1e-3
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=2,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    algo._adapt(samples)
    paths2 = sampler.obtain_samples()
    samples2 = proc.process_samples(paths2)
    algo.optimize_policy([samples, samples2], log=False)
    assert torch.isfinite(policy.theta).all() and np.isfinite(algo.last_stats['loss_after'])


@pytest.mark.parametrize('exploration', [False, True])
def test_vpg_maml_matches_oracle(exploration):
    """VPGMAML (ref meta_algos/vpg_maml.py): meta objective / gradient and the single TF1-Adam step."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.meta_algos import VPGMAML
    from promp_b200.samplers.device_data import SamplesData
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    M, N, Do, Da = 4, 180, 2, 2
    np.random.seed(4)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64))
    algo = VPGMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                   inner_type='log_likelihood', exploration=exploration)
    dims = (Do, Da, (64, 64))
    theta = policy.theta.cpu().numpy().copy()
    cpus, phases = [], []
    for s in range(2):
        c, p = _random_phase(torch, M, N, Do, Da, theta, 110 + s)
        rew = torch.randn(M, N, generator=torch.Generator().manual_seed(5 + s)) + torch.arange(M).view(-1, 1).float()
        p.rew.copy_(rew)
        keep = p.adv.clone()
        run_process_kernel(p, 0.99, 1.0, 1e-5, 1, True, False)
        p.adv = keep
        c = {k: v.double() for k, v in c.items()}
        r64 = rew.double()
        c['adj_avg_rewards'] = (r64 - r64.mean()) / (r64.std(unbiased=False) + 1e-8)
        cpus.append(c); phases.append(p)
    t64 = torch.tensor(theta, dtype=torch.float64, requires_grad=True)
    obj, _, _ = th.meta_objective(t64, cpus, dims, 0.1, 'vpg', inner_type='log_likelihood', exploration=exploration)
    (g_want,) = torch.autograd.grad(obj, t64)
    res = algo._objective_pass(phases, want_grad=True)
    assert rel_err(res['grad'].cpu().numpy(), g_want.numpy()) < 1e-4
    assert abs(float(algo.loss_terms(res)[0]) - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
    algo.optimize_policy([[SamplesData(p, m) for m in range(M)] for p in phases], log=False)
    adam = th.TF1Adam(theta.size)
    want = adam.step(torch.tensor(theta), g_want.float())
    np.testing.assert_allclose(policy.theta.cpu().numpy(), want.numpy(), rtol=0, atol=2e-5)
    assert abs(algo.last_stats['loss_before'] - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))


@pytest.mark.parametrize('Do,Da,N', [(2, 2, 2000), (17, 6, 700), (2, 2, 130), (4, 2, 391)])
def test_tensor_core_policy_grad_matches_simt_and_oracle(Do, Da, N):
    """promp_set_option("tensor_cores", 1): the tensor-core (mma.sync) 3xTF32 path of policy_grad (layer GEMMs on the tensor
    cores) gives the CUDA-core path's results to fp32 round-off, for shared and per-task parameters, grad and
    eval-only modes."""
    torch = _cuda()
    from promp_b200 import _lib
    from oracle import tf_half as th
    M = 7
    policy, algo = _algo(torch, 'promp', M, Do, Da)
    theta = policy.theta.cpu().numpy()
    cpu, ph = _random_phase(torch, M, N, Do, Da, theta, 8)
    P = policy.num_params
    theta_t = (policy.theta.view(1, -1) + 0.05 * torch.randn(M, P, generator=torch.Generator().manual_seed(3)).cuda()).contiguous()
    res = {}
    try:
        for tc in (0, 1, 2):          # 0: CUDA cores; 1 / 2: tensor-core path with 256 / 512 threads per CTA
            _lib.set_option('tensor_cores', 1 if tc else 0)
            _lib.set_option('tc_threads', {0: 0, 1: 256, 2: 512}[tc])
            out = []
            for params, stride in ((policy.theta, 0), (theta_t, P)):
                for obj in (0, 1, 2):
                    g = torch.empty(M, P, device='cuda'); newp = torch.empty(M, P, device='cuda'); st = torch.zeros(M, 4, device='cuda')
                    algo._grad(ph, params, stride, obj, clip_eps=0.3, kl_coeff=0.01, clip_log_std=1, grad=g, out_params=newp,
                               sgd_lr=0.1, stats=st)
                    st2 = torch.zeros(M, 4, device='cuda')
                    algo._grad(ph, params, stride, obj, clip_eps=0.3, kl_coeff=0.01, clip_log_std=1, stats=st2)   # eval only
                    out.append((g.cpu().numpy(), newp.cpu().numpy(), st.cpu().numpy(), st2.cpu().numpy()))
            res[tc] = out
    finally:
        _lib.set_option('tensor_cores', 1)
        _lib.set_option('tc_threads', 0)
    for tc in (1, 2):
        for a, b in zip(res[0], res[tc]):
            assert rel_err(b[0], a[0]) < 2e-5, rel_err(b[0], a[0])
            np.testing.assert_allclose(b[1], a[1], rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(b[2][:, :3], a[2][:, :3], rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(b[3][:, :3], a[2][:, :3], rtol=1e-5, atol=1e-6)
    # and against the fp64 oracle: the inner adapt step with shared theta, likelihood-ratio objective, no KL term
    try:
        _lib.set_option('tensor_cores', 1)
        g = torch.empty(M, P, device='cuda'); newp = torch.empty(M, P, device='cuda')
        algo._grad(ph, policy.theta, 0, 0, grad=g, out_params=newp, sgd_lr=0.1)
    finally:
        _lib.set_option('tensor_cores', 1)
    c64 = {k: v.double() for k, v in cpu.items()}
    want = th.adapt(torch.tensor(theta, dtype=torch.float64).view(1, -1).expand(M, -1).contiguous(), c64, (Do, Da, (64, 64)), 0.1)
    g_want = (torch.tensor(theta, dtype=torch.float64).view(1, -1) - want) / 0.1
    assert rel_err(g.cpu().numpy(), g_want.numpy()) < 1e-4


@pytest.mark.parametrize('Do,Da,N,stride_mode', [(2, 2, 2000, 'shared'), (2, 2, 2000, 'per_task'), (2, 2, 130, 'shared'),
                                                  (17, 6, 700, 'per_task'), (17, 6, 129, 'shared'), (4, 2, 391, 'per_task')])
def test_tensor_core_policy_hvp_matches_simt(Do, Da, N, stride_mode):
    """The tensor-core path of policy_hvp (forward and backward layer GEMMs as 3xTF32 MMAs with the "lo" A operands in
    tensor memory) gives the CUDA-core path's backward-chain vector to fp32 round-off, for both inner
    objectives, with and without the KL term, and with the log_std clip mask active."""
    torch = _cuda()
    from promp_b200 import _lib
    M = 7
    res = {}
    for inner in ('likelihood_ratio', 'log_likelihood'):
        policy, algo = _algo(torch, 'trpo', M, Do, Da, inner_type=inner)
        theta = policy.theta.cpu().numpy()
        cpu, ph = _random_phase(torch, M, N, Do, Da, theta, 11)
        P = policy.num_params
        gen = torch.Generator().manual_seed(5)
        theta_t = (policy.theta.view(1, -1) + 0.05 * torch.randn(M, P, generator=gen).cuda()).contiguous()
        vec = torch.randn(M, P, generator=gen).cuda().contiguous()
        params, stride = (policy.theta, 0) if stride_mode == 'shared' else (theta_t, P)
        try:
            for tc in (0, 1, 2):      # 0: CUDA cores; 1 / 2: tensor-core path with 256 / 512 threads per CTA
                _lib.set_option('tensor_cores', 1 if tc else 0)
                _lib.set_option('tc_threads', {0: 0, 1: 256, 2: 512}[tc])
                out = []
                for klc, clip in ((0.0, 0), (5e-3, 0), (5e-3, 1)):
                    hv = torch.empty(M, P, device='cuda'); st = torch.zeros(M, 4, device='cuda')
                    algo._hvp(ph, params, stride, vec, hv, klc, clip, stats=st)
                    out.append((hv.cpu().numpy(), st.cpu().numpy()))
                res[(inner, tc)] = out
        finally:
            _lib.set_option('tensor_cores', 1)
            _lib.set_option('tc_threads', 0)
        for tc in (1, 2):
            for a, b in zip(res[(inner, 0)], res[(inner, tc)]):
                d = rel_err(b[0] - vec.cpu().numpy(), a[0] - vec.cpu().numpy())      # compare the H v part, not v + ...
                assert d < 5e-5, d
                np.testing.assert_allclose(b[1][:, :3], a[1][:, :3], rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# variable-length paths (SURVEY.md section 8f item 2: early termination, meta_sampler.py:116-125)
@pytest.mark.parametrize('case', ['r1', 'r2', 'r3'])
def test_process_samples_ragged_matches_reference_golden(golden_dir, case):
    """MetaSampleProcessor on variable-length host paths -> promp_process_samples_ragged, against the unmodified
    reference's outputs (tests/golden/process_samples_ragged.npz): returns, baseline coefficients, advantages."""
    torch = _cuda()
    from test_oracle_golden import ragged_paths_from_golden
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    g = np.load(os.path.join(golden_dir, 'process_samples_ragged.npz'))
    pre = 'case_%s_' % case
    paths = ragged_paths_from_golden(g, pre)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=float(g[pre + 'cfg_discount']),
                               gae_lambda=float(g[pre + 'cfg_gae_lambda']), normalize_adv=bool(g[pre + 'cfg_normalize_adv']),
                               positive_adv=bool(g[pre + 'cfg_positive_adv']))
    data = proc.process_samples(paths, log=False)
    assert len(data) == len(paths) and len(data[0].keys()) == 8
    got_ret = np.concatenate([d['returns'] for d in data])
    got_adv = np.concatenate([d['advantages'] for d in data])
    np.testing.assert_allclose(got_ret, g[pre + 'returns'], rtol=2e-7, atol=1e-6)
    assert rel_err(got_adv, g[pre + 'advantages']) < 1e-5
    np.testing.assert_allclose(data[0].phase.host('coeffs'), g[pre + 'coeffs'], rtol=1e-6, atol=1e-8)
    np.testing.assert_array_equal(np.concatenate([d['observations'] for d in data]), g[pre + 'observations_stacked'])
    # sample counts per task follow the path table
    lens = np.split(g[pre + 'path_len'], np.cumsum(g[pre + 'n_paths'])[:-1])
    assert [len(d['rewards']) for d in data] == [int(l.sum()) for l in lens]


def _ragged_phase(torch, n_valid, Do, Da, theta, seed, paths_per_task=3):
    """Synthetic variable-length phase: task m has n_valid[m] samples split into a few paths; padding rows hold garbage
    on purpose (they must not contribute)."""
    from promp_b200.samplers.device_data import RaggedPhaseData
    from oracle import tf_half as th
    M = len(n_valid)
    g = torch.Generator().manual_seed(seed)
    lens = []
    for n in n_valid:
        cuts = sorted(set(int(x) for x in torch.randint(1, n, (paths_per_task - 1,), generator=g))) if n > paths_per_task else []
        edges = [0] + cuts + [n]
        lens.append([b - a for a, b in zip(edges[:-1], edges[1:])])
    ph = RaggedPhaseData(lens, Do, Da, torch.device('cuda'))
    N = ph.N
    obs = torch.randn(M, N, Do, generator=g)
    th_t = torch.as_tensor(theta).view(1, -1).expand(M, -1)
    mean, ls = th.dist_info(th_t, obs, (Do, Da, (64, 64)))
    old_mean = mean + 0.1 * torch.randn(M, N, Da, generator=g)
    old_ls = (ls + 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
    act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
    adv = torch.randn(M, N, generator=g)
    cpu = []
    for m, n in enumerate(n_valid):
        cpu.append(dict(obs=obs[m:m + 1, :n], act=act[m:m + 1, :n], adv=adv[m:m + 1, :n], mean=old_mean[m:m + 1, :n],
                        log_std=old_ls[m:m + 1, :n]))
        obs[m, n:] = 1e3; act[m, n:] = -50.0; adv[m, n:] = 1e4; old_mean[m, n:] = 7.0          # poison the padding
    ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0])
    ph.adv = adv.cuda()
    return cpu, ph


@pytest.mark.parametrize('Do,Da', [(2, 2), (17, 6)])
@pytest.mark.parametrize('tc', [0, 1])
def test_ragged_meta_gradient_matches_oracle(Do, Da, tc):
    """ProMP meta-gradient with a different number of valid samples per task and per phase (promp_policy_*_ragged):
    per-task means run over n_valid[m], padding rows are ignored.  Oracle: fp64 autograd per task on the trimmed data."""
    torch = _cuda()
    from promp_b200 import _lib
    from oracle import tf_half as th
    M = 5
    policy, algo = _algo(torch, 'promp', M, Do, Da)
    dims = (Do, Da, (64, 64))
    theta = policy.theta.cpu().numpy()
    nv = [[130, 517, 64, 1000, 333], [257, 90, 700, 128, 411]]
    cpus, phases = [], []
    for s in range(2):
        c, p = _ragged_phase(torch, nv[s], Do, Da, theta, 20 + s)
        cpus.append(c); phases.append(p)
    coeff = list(algo.inner_kl_coeff)
    g_want, obj_want = 0.0, 0.0
    for m in range(M):
        t64 = torch.tensor(theta, dtype=torch.float64, requires_grad=True)
        data_m = [{k: v.double() for k, v in cpus[s][m].items()} for s in range(2)]
        obj, _, _ = th.meta_objective(t64, data_m, dims, 0.1, 'promp', 0.3, coeff)
        (gm,) = torch.autograd.grad(obj, t64)
        g_want = g_want + gm.numpy() / M
        obj_want += float(obj) / M
    try:
        _lib.set_option('tensor_cores', tc)
        res = algo._objective_pass(phases, want_grad=True)
        terms = algo.loss_terms(res).cpu().numpy()
        g_got = res['grad'].cpu().numpy()
    finally:
        _lib.set_option('tensor_cores', 1)
    assert abs(terms[0] - obj_want) < 1e-4 * max(1.0, abs(obj_want))
    err = rel_err(g_got, g_want)
    assert err < 1e-4, err


def test_snapshot_and_resume(tmp_path):
    """meta_trainer.py:144-158 + utils/logger.py:376-396: Trainer.train() writes a joblib snapshot {itr, policy, env,
    baseline} from device state plus progress.csv with the reference's keys; Trainer.restore() on a fresh stack brings
    back parameters, Adam slots, KL coefficients and counters, and training continues at itr + 1."""
    torch = _cuda()
    import csv
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    M, E, H = 4, 3, 30

    def make(n_itr):
        env, policy, sampler, proc = _make_stack('point', M, E, H)
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=2, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=True)
        return policy, algo, Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=n_itr,
                                     num_inner_grad_steps=1)
    d = str(tmp_path / 'run')
    try:
        logger.configure(dir=d, format_strs=['csv', 'json'], snapshot_mode='last')
        policy, algo, trainer = make(2)
        trainer.train()
        snap_path = os.path.join(d, 'params.pkl')
        assert os.path.exists(snap_path)
        rows = list(csv.DictReader(open(os.path.join(d, 'progress.csv'))))
        assert len(rows) == 2 and rows[1]['Itr'] == '1' and 'Step_1-AverageReturn' in rows[0] and 'LossAfter' in rows[0]
        snap = logger.load_snapshot(snap_path)
        assert set(('itr', 'policy', 'env', 'baseline')) <= set(snap) and snap['itr'] == 1
        assert torch.equal(snap['policy'].theta.cpu(), policy.theta.cpu())
        assert snap['baseline']._coeffs is not None and np.isfinite(np.asarray(snap['baseline']._coeffs)).all()
        # resume on a fresh stack
        logger.configure(dir=str(tmp_path / 'run2'), format_strs=['json'], snapshot_mode='none')
        np.random.seed(77)
        policy2, algo2, trainer2 = make(3)
        assert not torch.equal(policy2.theta, policy.theta)
        assert trainer2.restore(snap_path) == 2
        assert torch.equal(policy2.theta, policy.theta)
        assert torch.equal(algo2.optimizer.m, algo.optimizer.m) and torch.equal(algo2.optimizer.v, algo.optimizer.v)
        assert int(algo2.optimizer.step.item()) == int(algo.optimizer.step.item()) == 4
        np.testing.assert_array_equal(algo2.inner_kl_coeff, algo.inner_kl_coeff)
        assert trainer2.sampler.total_timesteps_sampled == 2 * 2 * M * E * H
        trainer2.train()                                            # runs exactly iteration 2
        kv = logger.last_dump()
        assert kv['Itr'] == 2 and kv['n_timesteps'] == 3 * 2 * M * E * H and np.isfinite(kv['LossAfter'])
    finally:
        logger.reset()


def test_half_cheetah_rand_vel_surrogate():
    """HalfCheetahRandVelEnv (half_cheetah_rand_vel.py:13-40): tasks ~ U(0,3) from the numpy RNG, reward_run =
    -|forward_vel - goal|, env_infos {forward_vel, reward_run, reward_ctrl}; fused rollout and the vec-env step kernel
    against the surrogate's spec (oracle/cheetah_surrogate.py) replayed with the kernel's own actions; one full ProMP
    iteration through the Trainer with the reference's log keys."""
    torch = _cuda()
    from oracle import cheetah_surrogate as cs
    from promp_b200.envs import normalize, HalfCheetahRandVelEnv
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.samplers.vectorized_env_executor import MetaDeviceEnvExecutor
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    M, E, H = 3, 4, 40
    np.random.seed(11)
    env = normalize(HalfCheetahRandVelEnv())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=17, action_dim=6, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    np.random.seed(5)
    want_tasks = np.random.uniform(0.0, 3.0, (M,))
    np.random.seed(5)
    sampler.update_tasks()
    goals = sampler.vec_env.task_params_per_task.cpu().numpy()[:, 0]
    np.testing.assert_allclose(goals, want_tasks.astype(np.float32), rtol=0, atol=0)
    rng = np.random.RandomState(2)
    noise = rng.randn(M, E, H, 6).astype(np.float32)
    init = np.zeros((M, E, 18), dtype=np.float32)
    init[..., :9] = rng.uniform(-.1, .1, size=(M, E, 9))
    init[..., 9:] = 0.1 * rng.randn(M, E, 9)
    policy.switch_to_pre_update()
    sampler.inject(noise=noise, init_state=init)
    ph = sampler.obtain_samples().phase
    assert ph.info.shape[0] == 3 and ph.info_keys == ('reward_run', 'reward_ctrl', 'forward_vel')
    obs = ph.obs.cpu().numpy().reshape(M, E, H, 17)
    act = ph.act.cpu().numpy().reshape(M, E, H, 6)
    rew = ph.rew.cpu().numpy().reshape(M, E, H)
    info = ph.info.cpu().numpy().reshape(3, M, E, H)
    qpos, qvel = init[..., :9].copy(), init[..., 9:].copy()
    for t in range(H):
        u = np.clip(np.float32(-1.0) + (act[:, :, t] + np.float32(10.0)) * np.float32(2.0) / np.float32(20.0), -1, 1)
        x0 = qpos[..., 0].copy()
        qpos, qvel, r, rr, rc = cs.step(qpos, qvel, u.astype(np.float32), None, goal_velocity=goals[:, None].astype(np.float32))
        np.testing.assert_allclose(info[2, :, :, t], (qpos[..., 0] - x0) / np.float32(0.05), rtol=1e-3, atol=2e-4)
        np.testing.assert_allclose(info[0, :, :, t], rr, rtol=1e-3, atol=2e-4)
        np.testing.assert_allclose(info[0, :, :, t], -np.abs(info[2, :, :, t] - goals[:, None]), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(rew[:, :, t], r, rtol=1e-3, atol=2e-4)
        if t + 1 < H:
            qpos[..., 1:] = obs[:, :, t + 1, :8]
            qvel[...] = obs[:, :, t + 1, 8:]
    # vec-env step kernel: same reward mode, three env_infos keys
    ex = MetaDeviceEnvExecutor(env, 2, 1, max_path_length=10)
    ex.set_tasks([0.5, 2.5])
    ex.reset()
    _, r, d, infos = ex.step([np.ones(6), -np.ones(6)])
    assert set(infos[0]) == {'reward_run', 'reward_ctrl', 'forward_vel'}
    for i, goal in enumerate((0.5, 2.5)):
        assert abs(infos[i]['reward_run'] + abs(infos[i]['forward_vel'] - goal)) < 1e-5
        assert abs(r[i] - (infos[i]['reward_run'] + infos[i]['reward_ctrl'])) < 1e-5
    # one full iteration through the trainer
    logger.set_quiet(True)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=2)
    Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=1, num_inner_grad_steps=1).train()
    kv = logger.last_dump()
    assert np.isfinite(kv['LossAfter']) and 'Step_1-AvgForwardVel' in kv and np.isfinite(kv['Step_0-AverageReturn'])


def test_point_walls_and_momentum_envs(golden_dir):
    """MetaPointEnvWalls / MetaPointEnvMomentum (SURVEY.md section 8f item 3): the vec-env step kernel against the
    unmodified reference (tests/golden/point_variants_steps.npz, trajectory glued to the reference each step so float32
    drift cannot flip a wall decision later), task draws in the reference's RNG order, the fused rollout bit-identical to
    the step kernel, and a full ProMP iteration on the momentum env (obs_dim 4 policy kernels)."""
    torch = _cuda()
    from promp_b200.envs import normalize, MetaPointEnvWalls, MetaPointEnvMomentum
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor, MetaDeviceEnvExecutor
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    g = _load(golden_dir, 'point_variants_steps.npz')
    # ---- walls: tasks (RNG order) + steps
    T, n_env, _ = g['walls_actions'].shape
    for rtype in ('dense', 'dense_squared'):
        env = normalize(MetaPointEnvWalls(reward_type=rtype))
        np.random.seed(17)
        tasks = env.sample_tasks(n_env)
        np.testing.assert_array_equal(np.stack([np.concatenate([t['goal'], t['gap_1'], t['gap_2']]) for t in tasks]), g['walls_tasks'])
        ex = MetaDeviceEnvExecutor(env, n_env, 1, max_path_length=10 ** 6)
        ex.set_tasks(tasks)
        ex.state.copy_(torch.from_numpy(g['walls_obs0'].astype(np.float32)))
        n_bad = 0
        for t in range(T):
            obs, rew, dones, infos = ex.step(g['walls_actions'][t])
            want = g['walls_next_obs_' + rtype][t]
            bad = np.abs(np.asarray(obs) - want).max(axis=1) > 5e-5          # a float32 norm within 1 ulp of a wall radius
            n_bad += int(bad.sum())
            np.testing.assert_allclose(np.asarray(rew), g['walls_rewards_' + rtype][t], rtol=1e-5, atol=1e-5)
            assert not dones.any() and infos[0] == {}
            ex.state.copy_(torch.from_numpy(want.astype(np.float32)))
        assert n_bad <= 2, n_bad
    with pytest.raises(NotImplementedError):
        MetaPointEnvWalls(reward_type='sparse')
    # ---- momentum: steps for the three reward types
    T, n_env, _ = g['momentum_actions'].shape
    for rtype in ('sparse', 'dense', 'dense_squared'):
        env = normalize(MetaPointEnvMomentum(reward_type=rtype))
        np.random.seed(19)
        tasks = env.sample_tasks(n_env)
        np.testing.assert_array_equal(np.asarray(tasks, dtype=np.float64), g['momentum_goals'])
        ex = MetaDeviceEnvExecutor(env, n_env, 1, max_path_length=10 ** 6)
        ex.set_tasks(tasks)
        np.random.seed(19); env.sample_tasks(n_env)
        np.testing.assert_allclose(np.asarray(ex.reset()), g['momentum_obs0'], rtol=0, atol=1e-7)   # reset draw order: pos, vel per env
        for t in range(T):
            obs, rew, dones, infos = ex.step(g['momentum_actions'][t])
            np.testing.assert_allclose(np.asarray(obs), g['momentum_next_obs_' + rtype][t], rtol=0, atol=5e-5)
            np.testing.assert_allclose(np.asarray(rew), g['momentum_rewards_' + rtype][t], rtol=1e-4, atol=2e-5)
            ex.state.copy_(torch.from_numpy(g['momentum_next_obs_' + rtype][t].astype(np.float32)))
    # ---- fused rollout == step kernel replayed with the rollout's own actions (same device functions -> bit-identical)
    for make, sd in ((lambda: MetaPointEnvWalls(), 2), (lambda: MetaPointEnvMomentum(), 4)):
        M, E, H = 3, 4, 50
        np.random.seed(23)
        env = normalize(make())
        policy = MetaGaussianMLPPolicy(name="p", obs_dim=sd, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
        policy.set_params(policy.get_param_values() if False else policy.theta.cpu().numpy() * 3.0)     # larger actions: reach the walls
        sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
        sampler.update_tasks()
        policy.switch_to_pre_update()
        rng = np.random.RandomState(4)
        noise = (8.0 * rng.randn(M, E, H, 2)).astype(np.float32)
        init = np.zeros((M, E, sd), dtype=np.float32)
        init[..., :2] = rng.uniform(-0.2, 0.2, size=(M, E, 2))
        if sd == 4:
            init[..., 2:] = rng.uniform(-0.1, 0.1, size=(M, E, 2))
        sampler.inject(noise=noise, init_state=init)
        ph = sampler.obtain_samples().phase
        obs = ph.obs.cpu().numpy().reshape(M * E, H, sd)
        act = ph.act.cpu().numpy().reshape(M * E, H, 2)
        rew = ph.rew.cpu().numpy().reshape(M * E, H)
        assert np.isfinite(obs).all() and (sd == 4 or np.linalg.norm(obs, axis=-1).max() > 1.0)
        ex = MetaDeviceEnvExecutor(env, M, E, max_path_length=10 ** 6)
        ex.set_tasks(sampler.vec_env.tasks)
        ex.state.copy_(torch.from_numpy(init.reshape(M * E, sd)))
        for t in range(H):
            np.testing.assert_array_equal(ex.state.cpu().numpy(), obs[:, t])
            o, r, _, _ = ex.step(act[:, t])
            np.testing.assert_array_equal(np.asarray(r, dtype=np.float32), rew[:, t])
    # ---- a full ProMP iteration on the momentum env through the Trainer
    logger.set_quiet(True)
    np.random.seed(2)
    M, E, H = 4, 5, 30
    env = normalize(MetaPointEnvMomentum())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=4, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=2)
    th0 = policy.theta.clone()
    Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=1, num_inner_grad_steps=1).train()
    kv = logger.last_dump()
    assert np.isfinite(kv['LossAfter']) and np.isfinite(kv['Step_1-AverageReturn']) and not torch.equal(policy.theta, th0)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('Do,Da,M,N,S1', [(2, 2, 40, 2000, 1), (17, 6, 40, 4000, 1), (2, 2, 10, 2000, 1), (2, 2, 3, 130, 1),
                                          (2, 2, 7, 700, 2), (4, 2, 5, 391, 1)])
def test_dataflow_chain_matches_separate_launches(Do, Da, M, N, S1):
    """promp_policy_chain (inner gradients -> outer gradient -> HVP chain as ONE persistent dataflow launch with per-task ready
    flags) against the same stages as stand-alone launches, at the BASELINE.json sizes (configs[1] 40x2000, configs[2] 40x4000,
    configs[3] 10 tasks per GPU) and at ragged-edge sizes.  Same kernels' tile code, different partition of the per-task sums:
    equal to float32 summation noise; the chain itself is bitwise run-to-run deterministic and leaves its control words zero."""
    torch = _cuda()
    policy, algo = _algo(torch, 'promp', M, Do, Da, 64, S1=S1)
    theta = policy.theta.cpu().numpy()
    phases = [_random_phase(torch, M, N, Do, Da, theta, 20 + s, 64)[1] for s in range(S1 + 1)]

    from promp_b200 import _lib

    def run(chain, want_grad=True):
        algo.use_chain = chain
        _lib.set_option('chain', 1)          # force the dataflow kernel (the default picks it for short stages only)
        try:
            res = algo._objective_pass(phases, want_grad=want_grad, reduce=False)
            torch.cuda.synchronize()
        finally:
            _lib.set_option('chain', -1)
        return (res['grad_tasks'].clone() if want_grad else None), res['stats_all'].clone()
    g_ref, st_ref = run(False)
    g1, st1 = run(True)
    g2, st2 = run(True)
    assert torch.equal(g1, g2) and torch.equal(st1, st2), "dataflow chain is not run-to-run deterministic"
    assert torch.isfinite(g1).all()
    for m in range(M):
        e = rel_err(g1[m].cpu().numpy(), g_ref[m].cpu().numpy())
        assert e < 2e-5, (m, e)
    np.testing.assert_allclose(st1[:, :, :3].cpu().numpy(), st_ref[:, :, :3].cpu().numpy(), rtol=2e-5, atol=1e-6)
    # values-only chain (the statistics pass after the last Adam epoch)
    _, st3 = run(True, want_grad=False)
    np.testing.assert_allclose(st3[:, :, :3].cpu().numpy(), st_ref[:, :, :3].cpu().numpy(), rtol=2e-5, atol=1e-6)
    ctrl = algo._ws_chain[:4 + 2 * 6 * M].cpu().numpy()
    assert (ctrl == 0).all(), "control words (queue, finished-CTA count, ready flags, arrival counters) must be left zero"


@pytest.mark.parametrize('target', [1e3, 1e-12])
def test_adaptive_kl_coefficient_on_device_matches_host_rule(target):
    """ProMP(adaptive_inner_kl_penalty=True) - the reference class default (pro_mp.py:40, 201-214): the CUDA-graph Trainer applies
    the halve / double rule on the device (promp_adapt_kl_coeff), the eager path on the host like the reference.  Same seeds ->
    the same coefficient sequence, logged KLCoeffInner and parameters.  target 1e3: the inner KL is below target / 1.5 (halve
    every iteration); 1e-12: above target * 1.5 (double every iteration) - decisions that do not depend on the action noise, which
    the two modes draw from differently keyed Philox streams."""
    torch = _cuda()
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    logger.set_quiet(True)
    M, E, H, n_itr = 6, 5, 40, 4

    def run(graph):
        env, policy, sampler, proc = _make_stack('point', M, E, H, seed=5)
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                     clip_eps=0.3, target_inner_step=target, init_inner_kl_penalty=1e-2, adaptive_inner_kl_penalty=True)
        trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=n_itr,
                          num_inner_grad_steps=1, use_cuda_graph=graph)
        assert trainer.graph_capturable()                 # adaptive KL no longer forces the eager path
        step = trainer.capture_graph(warmup=2, log=True) if graph else None
        np.random.seed(77)
        logged = []
        for itr in range(n_itr):
            if graph:
                step(itr)
            else:
                trainer.train_iteration(itr, log=True)
            logged.append(float(dict(logger.getkvs())['KLCoeffInner']))
            logger.dumpkvs()
        return policy.theta.clone(), logged, np.array(algo.inner_kl_coeff, dtype=np.float64)
    th_g, log_g, c_g = run(True)
    th_e, log_e, c_e = run(False)
    factor = 0.5 if target == 1e3 else 2.0
    want = [1e-2 * factor ** (i + 1) for i in range(n_itr)]
    np.testing.assert_allclose(log_e, want, rtol=1e-6)          # the host rule did what the case is built to do
    np.testing.assert_allclose(log_g, log_e, rtol=1e-6)
    np.testing.assert_allclose(c_g, c_e, rtol=1e-6)
    assert torch.isfinite(th_g).all() and torch.isfinite(th_e).all()
    # (the two modes draw their action noise from differently keyed Philox streams, so the parameters themselves differ)
    # the kernels read the coefficient from the device: same meta-gradient, bit for bit, as with the host value
    policy, algo = _algo(torch, 'promp', 4, 2, 2, 64, S1=1)
    theta = policy.theta.cpu().numpy()
    phases = [_random_phase(torch, 4, 300, 2, 2, theta, 40 + s_, 64)[1] for s_ in range(2)]
    algo.inner_kl_coeff = np.array([3e-3])
    g_host = algo._objective_pass(phases, want_grad=True)['grad'].clone()
    live = algo._device_coeffs()
    g_dev = algo._objective_pass(phases, want_grad=True)['grad'].clone()
    assert torch.equal(g_host, g_dev)
    live.mul_(2.0)                                             # what promp_adapt_kl_coeff does in place
    g_dev2 = algo._objective_pass(phases, want_grad=True)['grad'].clone()
    assert not torch.equal(g_dev2, g_dev) and float(algo.inner_kl_coeff[0]) == pytest.approx(6e-3, rel=1e-6)
    algo._coeff_live = None
    algo.inner_kl_coeff = np.array([6e-3])
    assert torch.equal(algo._objective_pass(phases, want_grad=True)['grad'], g_dev2)
