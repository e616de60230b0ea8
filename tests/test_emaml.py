"""E-MAML (TRPOMAML / VPGMAML with exploration=True, ref meta_algos/trpo_maml.py:137-144) on every sampling path:
the device coefficient promp_emaml_coeff, the PROMP_OBJ_EXPLORE objective of the policy kernels, the exploration stage of
promp_policy_chain, variable-length paths end to end against the float64 oracle, CUDA-graph replay and sharded totals.

CPU tests check the ABI mirror; everything else needs an H100 (pytest -m gpu)."""
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIN_LOG_STD = math.log(1e-6)


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


# ------------------------------------------------------------------------------------------------ CPU
def test_explore_objective_kind_mirrors_header():
    from promp_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'promp_b200.h')) as f:
        header = f.read()
    assert int(re.search(r'PROMP_OBJ_EXPLORE\s*=\s*(\d+)', header).group(1)) == _lib.OBJ_EXPLORE == 4
    for name in ('promp_emaml_coeff', 'promp_emaml_totals', 'promp_emaml_finish', 'promp_reduce_tasks2'):
        assert name in _lib.EXPORTED_SYMBOLS and re.search(r'\bint %s\(' % name, header), name


def test_emaml_algorithms_are_graph_capturable():
    """TRPOMAML(exploration=True) no longer opts out of CUDA-graph replay (the Trainer still keeps early-terminating envs
    eager); the formula the device coefficient implements, in float64 numpy, is the reference's over valid samples."""
    from promp_b200.meta_algos import TRPOMAML
    assert TRPOMAML.graph_capturable.fget(object()) is True
    rng = np.random.RandomState(0)
    rews = [rng.randn(n) + m for m, n in enumerate([5, 1, 17])]
    c = _coeff_numpy(rews)
    allr = np.concatenate(rews)
    adj = (allr - allr.mean()) / (allr.std() + 1e-8)          # meta_sample_processor.py:40-44
    offs = np.cumsum([0] + [len(r) for r in rews])
    np.testing.assert_allclose(c, [adj[a:b].mean() for a, b in zip(offs[:-1], offs[1:])], rtol=1e-12)


def _coeff_numpy(rews):
    """c_m = (mean r_m - mean r_all) / (std r_all + 1e-8) over each task's valid rewards, float64."""
    allr = np.concatenate([np.asarray(r, dtype=np.float64) for r in rews])
    mu, sd = allr.mean(), allr.std()
    return np.array([(np.mean(np.asarray(r, dtype=np.float64)) - mu) / (sd + 1e-8) for r in rews])


# ------------------------------------------------------------------------------------------------ helpers (GPU)
def _policy(M, Do, Da, act='tanh', seed=1):
    from promp_b200.policies import MetaGaussianMLPPolicy
    np.random.seed(seed)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64),
                                   hidden_nonlinearity=act)
    th_l = policy.unpad_flat(policy.theta.cpu().numpy()).copy()
    th_l += 0.1 * np.random.RandomState(9).randn(th_l.size).astype(np.float32)
    policy.set_params(th_l)
    return policy


def _dist(theta, obs, dims, act, min_log_std=None):
    """The policy forward of oracle.tf_half with either hidden activation (float64 autograd)."""
    import torch
    from oracle import tf_half as th
    W0, b0, W1, b1, W2, b2, ls = th.split_params(theta, *dims)
    f = torch.tanh if act == 'tanh' else torch.relu
    h = f(torch.matmul(obs, W0) + b0.unsqueeze(-2))
    h = f(torch.matmul(h, W1) + b1.unsqueeze(-2))
    mean = torch.matmul(h, W2) + b2.unsqueeze(-2)
    if min_log_std is not None:
        ls = torch.clamp(ls, min=min_log_std)
    return mean, ls


def _fixed_phase(torch, M, N, Do, Da, th_l, seed, with_rewards=True):
    from promp_b200.samplers.device_data import PhaseData
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    from oracle import tf_half as th
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(M, N, Do, generator=g)
    mean, ls = th.dist_info(torch.as_tensor(th_l).view(1, -1).expand(M, -1), obs, (Do, Da, (64, 64)))
    old_mean = mean + 0.1 * torch.randn(M, N, Da, generator=g)
    old_ls = (ls + 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
    act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
    ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
    ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0])
    rew = torch.randn(M, N, generator=g) + 0.5 * torch.arange(M).view(-1, 1).float()
    if with_rewards:
        ph.rew.copy_(rew)
        run_process_kernel(ph, 0.99, 1.0, 1e-5, 1, True, False)
    cpu = dict(obs=obs.double(), act=act.double(), mean=old_mean.double(), log_std=old_ls.double(), rew=rew.double())
    return cpu, ph


def _ragged_phase(torch, path_lens, Do, Da, th_l, seed):
    """Variable-length phase with poison in the padding rows, processed by the ragged kernel."""
    from promp_b200.samplers.device_data import RaggedPhaseData
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    from oracle import tf_half as th
    M = len(path_lens)
    ph = RaggedPhaseData(path_lens, Do, Da, torch.device('cuda'))
    N = ph.N
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(M, N, Do, generator=g)
    mean, ls = th.dist_info(torch.as_tensor(th_l).view(1, -1).expand(M, -1), obs, (Do, Da, (64, 64)))
    old_mean = mean + 0.1 * torch.randn(M, N, Da, generator=g)
    old_ls = (ls + 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
    act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
    rew = torch.randn(M, N, generator=g) + 0.5 * torch.arange(M).view(-1, 1).float()
    nv = [sum(l) for l in path_lens]
    for m, n in enumerate(nv):
        obs[m, n:] = 1e3; act[m, n:] = -50.0; old_mean[m, n:] = 7.0; rew[m, n:] = 1e4
    ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0]); ph.rew.copy_(rew)
    run_process_kernel(ph, 0.99, 1.0, 1e-5, 1, True, False)
    cpu = [dict(obs=obs[m:m + 1, :n].double(), act=act[m:m + 1, :n].double(), mean=old_mean[m:m + 1, :n].double(),
                log_std=old_ls[m:m + 1, :n].double(), rew=rew[m, :n].double()) for m, n in enumerate(nv)]
    return cpu, ph


def _trpo(policy, M, S1=1, **kw):
    from promp_b200.meta_algos import TRPOMAML
    return TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, step_size=0.01, exploration=True,
                    **kw)


# ------------------------------------------------------------------------------------------------ 1. coefficient
@pytest.mark.gpu
@pytest.mark.parametrize('M,N', [(5, 300), (40, 2000), (3, 1)])
def test_coefficient_fixed_horizon_matches_eager_path_bit_for_bit(M, N):
    torch = _cuda()
    policy = _policy(M, 2, 2)
    algo = _trpo(policy, M)
    cpu, ph = _fixed_phase(torch, M, N, 2, 2, policy.unpad_flat(policy.theta.cpu().numpy()), 7)
    phases = [ph, ph]
    c = algo.exploration_coeff_dev(phases)
    old = algo._exploration_coeff(phases)
    assert old.shape == (M, N) and c.shape == (M,) and c.dtype == torch.float32
    assert torch.equal(c, old[:, 0]), (c, old[:, 0])
    want = _coeff_numpy([cpu['rew'][m].numpy() for m in range(M)])
    np.testing.assert_allclose(c.cpu().numpy(), want, rtol=1e-6, atol=1e-7)
    assert algo.exploration_coeff_dev(phases) is c                    # once per phase and data generation
    # against the adj_avg_rewards the sample processor hands out (the reference's sample key)
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    MetaSampleProcessor(baseline=LinearFeatureBaseline()).compute_adj_avg_rewards(ph)
    np.testing.assert_allclose(c.cpu().numpy(), ph.adj_avg_rewards.double().mean(1).cpu().numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_coefficient_variable_length_matches_reference_formula():
    """Means over each task's valid samples, including a task with one short path (3 samples) and one with a single
    sample; the poisoned padding rows never enter."""
    torch = _cuda()
    path_lens = [[40, 17, 60], [3], [1], [100, 100, 25, 9], [7, 8]]
    policy = _policy(len(path_lens), 2, 2)
    algo = _trpo(policy, len(path_lens))
    cpu, ph = _ragged_phase(torch, path_lens, 2, 2, policy.unpad_flat(policy.theta.cpu().numpy()), 3)
    c = algo.exploration_coeff_dev([ph, ph]).cpu().numpy()
    want = _coeff_numpy([d['rew'].numpy() for d in cpu])
    np.testing.assert_allclose(c, want, rtol=1e-6, atol=1e-7)
    # the eager statement stays fixed-horizon only
    with pytest.raises(NotImplementedError):
        algo._exploration_coeff([ph, ph])
    # the three entry points agree: totals + finish on this launch's own totals == promp_emaml_coeff
    from promp_b200 import _lib
    tot = torch.empty(3, dtype=torch.float64, device='cuda')
    c2 = torch.empty(ph.M, dtype=torch.float32, device='cuda')
    _lib.call('promp_emaml_totals', ph.M, _lib.ptr(ph.stats), _lib.ptr(ph.n_valid), ph.N, _lib.ptr(tot), _lib.stream())
    _lib.call('promp_emaml_finish', ph.M, _lib.ptr(ph.stats), _lib.ptr(ph.n_valid), ph.N, _lib.ptr(tot), _lib.ptr(c2), _lib.stream())
    assert np.array_equal(c2.cpu().numpy(), c)
    assert float(tot[2]) == sum(sum(l) for l in path_lens)
    with pytest.raises(_lib.PrompLibraryError):
        _lib.call('promp_emaml_coeff', 0, _lib.ptr(ph.stats), None, 5, _lib.ptr(c2), _lib.stream())


@pytest.mark.gpu
@pytest.mark.parametrize('W', [2, 4])
def test_coefficient_of_shards_equals_one_process(W, monkeypatch):
    """The rank path of exploration_coeff_dev (totals -> sum over ranks -> finish) on slices of one global phase: each
    rank's tasks are processed on their own, and the exchange is replaced by the sum of every shard's totals.  Equal to
    one process with the global batch.  This checks the arithmetic of the split; that sharded rollouts feed the same
    per-task reward sums is checked by test_coefficient_of_sharded_sampling_equals_one_process."""
    torch = _cuda()
    import promp_b200.meta_algos.trpo_maml as tm
    from promp_b200.samplers.device_data import PhaseData
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    M, N = 8 * W, 500
    policy = _policy(M, 2, 2)
    algo = _trpo(policy, M)
    _, glob = _fixed_phase(torch, M, N, 2, 2, policy.unpad_flat(policy.theta.cpu().numpy()), 11)
    want = algo.exploration_coeff_dev([glob, glob]).clone()
    Ml = M // W
    shards = []
    for r in range(W):
        ph = PhaseData(Ml, 1, N, 2, 2, torch.device('cuda'))
        ph.obs.copy_(glob.obs[r * Ml:(r + 1) * Ml]); ph.rew.copy_(glob.rew[r * Ml:(r + 1) * Ml])
        run_process_kernel(ph, 0.99, 1.0, 1e-5, 1, True, False)
        assert torch.equal(ph.stats, glob.stats[r * Ml:(r + 1) * Ml])
        shards.append(ph)
    from promp_b200 import _lib
    totals = []
    for ph in shards:
        t = torch.empty(3, dtype=torch.float64, device='cuda')
        _lib.call('promp_emaml_totals', Ml, _lib.ptr(ph.stats), None, N, _lib.ptr(t), _lib.stream())
        totals.append(t)
    summed = sum(totals[1:], totals[0].clone())
    monkeypatch.setattr(tm, 'world_size', lambda: W)
    monkeypatch.setattr(tm, 'allreduce_sum_', lambda t: t.copy_(summed))
    got = []
    for ph in shards:
        alg = _trpo(_policy(Ml, 2, 2), Ml)
        got.append(alg.exploration_coeff_dev([ph, ph]))
    got = torch.cat(got)
    np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-6, atol=1e-7)
    n_equal = int((got == want).sum())
    assert n_equal >= M - 1, "float64 totals summed per shard may differ from the global order only in the last bit"


@pytest.mark.gpu
@pytest.mark.parametrize('reset_mode', ['numpy', 'device'])
def test_coefficient_of_sharded_sampling_equals_one_process(reset_mode, monkeypatch):
    """MetaSampler(task_shard=(r, 2)) run one rank after another on one GPU, with the same numpy and Philox seeds as one
    process with the global batch (cheetah surrogate, fixed horizon): each rank's phase is sampled and processed, and its
    coefficient goes through the rank path with the exchange replaced by the sum of both ranks' totals.  The two ranks'
    coefficients together equal the one-process coefficient."""
    torch = _cuda()
    import promp_b200.meta_algos.trpo_maml as tm
    from promp_b200 import _lib
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, HalfCheetahRandDirecEnv
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    W, MG, E, H = 2, 8, 5, 37

    def phase(M, shard):
        np.random.seed(21)
        env = normalize(HalfCheetahRandDirecEnv())
        Do, Da = int(np.prod(env.observation_space.shape)), int(np.prod(env.action_space.shape))
        policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64))
        sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                              reset_mode=reset_mode, seed=5, task_shard=shard)
        np.random.seed(22)
        sampler.update_tasks()
        policy.switch_to_pre_update()
        proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
        return policy, proc.process_samples(sampler.obtain_samples())[0].phase
    policy, glob = phase(MG, None)
    want = _trpo(policy, MG).exploration_coeff_dev([glob, glob]).clone()
    shards = [phase(MG // W, (r, W)) for r in range(W)]
    for r, (_, ph) in enumerate(shards):
        assert torch.equal(ph.rew, glob.rew[r * (MG // W):(r + 1) * (MG // W)])
    totals = []
    for _, ph in shards:
        t = torch.empty(3, dtype=torch.float64, device='cuda')
        _lib.call('promp_emaml_totals', ph.M, _lib.ptr(ph.stats), None, ph.N, _lib.ptr(t), _lib.stream())
        totals.append(t)
    summed = totals[0] + totals[1]
    monkeypatch.setattr(tm, 'world_size', lambda: W)
    monkeypatch.setattr(tm, 'allreduce_sum_', lambda t: t.copy_(summed))
    got = torch.cat([_trpo(pol, ph.M).exploration_coeff_dev([ph, ph]) for pol, ph in shards])
    np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------------------------------------ 2. objective
CASES = [(2, 2, 300), (17, 6, 200), (3, 1, 130), (11, 5, 257)]      # exact (2,2), (17,6); padded (3,1) and (11,5)


@pytest.mark.gpu
@pytest.mark.parametrize('act', ['tanh', 'relu'])
@pytest.mark.parametrize('Do,Da,N', CASES)
@pytest.mark.parametrize('tc', [1, 0])
def test_explore_objective_matches_autograd(Do, Da, N, act, tc):
    """PROMP_OBJ_EXPLORE: value -c_m * mean log pi_theta(a|x) (clipped log_std) and its gradient per task and per parameter
    block against float64 autograd; on fixed-horizon data it equals the LOGLIK objective on the expanded [M, N] weights."""
    torch = _cuda()
    from promp_b200 import _lib
    from oracle import tf_half as th
    M = 5
    policy = _policy(M, Do, Da, act)
    algo = _trpo(policy, M)
    th_l = policy.unpad_flat(policy.theta.cpu().numpy())
    cpu, ph = _fixed_phase(torch, M, N, Do, Da, th_l, 5)
    c = torch.tensor([0.7, -1.3, 0.0, 2.1, -0.4], dtype=torch.float32, device='cuda')
    P = policy.num_params
    _lib.set_option('tensor_cores', tc)
    try:
        g = torch.empty(M, P, device='cuda'); st = torch.empty(M, 4, device='cuda')
        algo._grad(ph, policy.theta, 0, _lib.OBJ_EXPLORE, clip_log_std=1, grad=g, stats=st, adv=c)
        g_old = torch.empty(M, P, device='cuda'); st_old = torch.empty(M, 4, device='cuda')
        algo._grad(ph, policy.theta, 0, _lib.OBJ_LOGLIK, clip_log_std=1, grad=g_old, stats=st_old,
                   adv=c.view(-1, 1).expand(M, N).contiguous())
        torch.cuda.synchronize()
    finally:
        _lib.set_option('tensor_cores', 1)
    dims = (Do, Da, (64, 64))
    t64 = torch.tensor(th_l, dtype=torch.float64, requires_grad=True)
    mean, ls = _dist(t64.unsqueeze(0).expand(M, -1), cpu['obs'], dims, act, MIN_LOG_STD)
    val = -c.double().cpu() * th.log_likelihood(cpu['act'], mean, ls).mean(-1)
    val_np = val.detach().numpy()
    shapes = list(th.param_shapes(Do, Da).values())
    offs = np.cumsum([0] + [int(np.prod(s)) for s in shapes])
    for m in range(M):
        assert abs(float(st[m, 0]) - val_np[m]) <= 1e-4 * max(1.0, abs(val_np[m])), m
        (gm,) = torch.autograd.grad(val[m], t64, retain_graph=True)
        got = policy.unpad_flat(g[m].cpu().numpy())
        for b in range(len(shapes)):
            want = gm[offs[b]:offs[b + 1]].numpy()
            if np.linalg.norm(want) == 0.0:
                assert np.abs(got[offs[b]:offs[b + 1]]).max() == 0.0, (m, b)
            else:
                assert rel_err(got[offs[b]:offs[b + 1]], want) < 1e-4, (m, b)
    pad = np.ones(P, dtype=bool)                           # _pad_index_np: where the logical parameters sit
    pad[policy._pad_index_np] = False
    assert (g.cpu().numpy()[:, pad] == 0).all()            # zero-padded parameters get exactly zero gradient
    # the old path: the same objective with c materialised per sample
    assert rel_err(g.cpu().numpy(), g_old.cpu().numpy()) <= 1e-6
    np.testing.assert_allclose(st[:, 0].cpu().numpy(), st_old[:, 0].cpu().numpy(), rtol=1e-6, atol=1e-7)


@pytest.mark.gpu
def test_explore_objective_variable_length_and_argument_checks():
    torch = _cuda()
    from promp_b200 import _lib
    from oracle import tf_half as th
    path_lens = [[40, 17, 60], [3], [1], [100, 100, 25, 9], [129]]
    M = len(path_lens)
    policy = _policy(M, 2, 2)
    algo = _trpo(policy, M)
    th_l = policy.unpad_flat(policy.theta.cpu().numpy())
    cpu, ph = _ragged_phase(torch, path_lens, 2, 2, th_l, 9)
    c = torch.tensor([0.5, -1.0, 2.0, 0.25, -0.75], dtype=torch.float32, device='cuda')
    g = torch.empty(M, policy.num_params, device='cuda'); st = torch.empty(M, 4, device='cuda')
    algo._grad(ph, policy.theta, 0, _lib.OBJ_EXPLORE, clip_log_std=1, grad=g, stats=st, adv=c)
    t64 = torch.tensor(th_l, dtype=torch.float64, requires_grad=True)
    for m, d in enumerate(cpu):
        mean, ls = th.dist_info(t64.unsqueeze(0), d['obs'], (2, 2, (64, 64)), MIN_LOG_STD)
        v = -float(c[m]) * th.log_likelihood(d['act'], mean, ls).mean()
        (gm,) = torch.autograd.grad(v, t64)
        v = v.item()
        assert abs(float(st[m, 0]) - v) <= 1e-4 * max(1.0, abs(v))
        assert rel_err(g[m].cpu().numpy(), gm.numpy()) < 1e-4, m
    # the HVP entry points take RATIO / LOGLIK only; a chain's EXPLORE stage must be the last one
    ws = algo._workspace(ph.N)
    with pytest.raises(_lib.PrompLibraryError):
        _lib.call('promp_policy_hvp_ragged', 2, 2, 64, M, ph.N, _lib.ptr(ph.n_valid), _lib.ptr(policy.theta), 0, _lib.ptr(ph.obs),
                  _lib.ptr(ph.act), _lib.ptr(c), _lib.ptr(ph.mean), _lib.ptr(ph.log_std), 0, _lib.OBJ_EXPLORE, 0.1, 0.0, 1,
                  MIN_LOG_STD, _lib.ptr(g), _lib.ptr(g), None, _lib.ptr(ws), ws.numel() * 4, _lib.stream())
    st_x = algo._stage(0, ph, policy.theta, 0, _lib.OBJ_EXPLORE, clip_log_std=1, grad=g, stats=st, adv=c)
    st_o = algo._stage(0, ph, policy.theta, 0, _lib.OBJ_LOGLIK, clip_log_std=1, grad=g, stats=st)
    with pytest.raises(_lib.PrompLibraryError):
        algo._run_chain([st_x, st_o])


# ------------------------------------------------------------------------------------------------ 3. ragged end to end
def _device_ragged_phases(torch, env_name, algo_name, M=6, E=4, H=60, seed=4):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnv, Walker2DRandVelEnv
    from promp_b200.meta_algos import VPGMAML
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    np.random.seed(seed)
    torch.manual_seed(seed)
    env = normalize(MetaPointEnv() if env_name == 'point' else Walker2DRandVelEnv())
    Do, Da = int(np.prod(env.observation_space.shape)), int(np.prod(env.action_space.shape))
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          reset_mode='device')
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    if algo_name == 'trpo':
        algo = _trpo(policy, M)
    else:
        algo = VPGMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                       inner_type='log_likelihood', exploration=True)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    samples = []
    for step in range(2):
        s = proc.process_samples(sampler.obtain_samples())
        samples.append(s)
        if step == 0:
            algo._adapt(s)
    return policy, algo, samples, (Do, Da, (64, 64))


@pytest.mark.gpu
@pytest.mark.parametrize('env_name', ['point', 'walker'])
@pytest.mark.parametrize('algo_name', ['trpo', 'vpg'])
def test_ragged_emaml_matches_oracle(env_name, algo_name):
    """TRPOMAML / VPGMAML(exploration=True) on device-sampled variable-length paths (reset_mode='device'): meta-objective, KL
    terms and gradient against oracle.tf_half on the same float32 samples, each task fed its valid samples only."""
    torch = _cuda()
    from oracle import tf_half as th
    policy, algo, samples, dims = _device_ragged_phases(torch, env_name, algo_name, H=60 if env_name == 'point' else 200)
    M = algo.meta_batch_size
    phases = [algo._phase_of(s) for s in samples]
    assert all(getattr(p, 'n_valid', None) is not None for p in phases)
    if env_name == 'walker':                                  # some paths ended early (the walker fell)
        assert int(phases[1].n_paths.sum()) > M * 4
    c_want = _coeff_numpy([np.asarray(samples[1][m]['rewards']) for m in range(M)])
    np.testing.assert_allclose(algo.exploration_coeff_dev(phases).cpu().numpy(), c_want, rtol=1e-6, atol=1e-7)

    def task_dict(s, m, with_adj):
        d = dict(obs=s['observations'], act=s['actions'], adv=s['advantages'], mean=s['agent_infos']['mean'],
                 log_std=s['agent_infos']['log_std'])
        d = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)).unsqueeze(0) for k, v in d.items()}
        if with_adj:
            d['adj_avg_rewards'] = torch.tensor([[c_want[m]]], dtype=torch.float64)
        return d
    t64 = torch.tensor(policy.theta.cpu().numpy(), dtype=torch.float64, requires_grad=True)
    kind = 'trpo' if algo_name == 'trpo' else 'vpg'
    inner = 'likelihood_ratio' if algo_name == 'trpo' else 'log_likelihood'
    objs, ikls, okls = [], [], []
    for m in range(M):
        o, ik, ok = th.meta_objective(t64, [task_dict(samples[0][m], m, False), task_dict(samples[1][m], m, True)], dims, 0.1,
                                      kind, inner_type=inner, exploration=True)
        objs.append(o); ikls.append(ik[0]); okls.append(ok)
    obj, ikl, okl = torch.stack(objs).mean(), torch.stack(ikls).mean(), torch.stack(okls).mean()
    (g_want,) = torch.autograd.grad(obj, t64)
    obj, ikl, okl = obj.item(), ikl.item(), okl.item()
    if algo_name == 'trpo':
        terms = algo.loss_terms_dev(policy.theta, phases).cpu().numpy()
        g_got = algo.eval_gradient(policy.theta, phases, 'loss')
    else:
        res = algo._objective_pass(phases, want_grad=True)
        terms = algo.loss_terms(res).cpu().numpy()
        g_got = res['grad'].cpu().numpy()
    for got, want in zip(terms, (obj, ikl, okl)):
        assert abs(float(got) - float(want)) <= 1e-4 * max(1.0, abs(float(want))), (terms, float(obj), float(ikl), float(okl))
    assert rel_err(g_got, g_want.numpy()) < 1e-4
    # the exploration term is exercised: without it the objective differs
    plain = torch.stack([th.meta_objective(t64, [task_dict(samples[0][m], m, False), task_dict(samples[1][m], m, False)],
                                           dims, 0.1, kind, inner_type=inner)[0] for m in range(M)]).mean()
    assert abs(plain.item() - obj) > 1e-6


@pytest.mark.gpu
def test_ragged_emaml_optimize_policy_runs():
    """One TRPO-MAML E-MAML outer step on device-sampled walker paths: finite, parameters move."""
    torch = _cuda()
    from promp_b200.utils import logger
    logger.set_quiet(True)
    policy, algo, samples, _ = _device_ragged_phases(torch, 'walker', 'trpo')
    th0 = policy.theta.clone()
    algo.optimize_policy(samples, log=False)
    assert torch.isfinite(policy.theta).all() and not torch.equal(policy.theta, th0)
    assert all(np.isfinite(v) for v in algo.last_stats.values())


# ------------------------------------------------------------------------------------------------ 4. chain
@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,M,N,S1', [(2, 2, 40, 2000, 1), (17, 6, 20, 1000, 1), (2, 2, 7, 700, 2), (2, 2, 3, 130, 1)])
def test_chain_with_exploration_stage_matches_separate_launches(Do, Da, M, N, S1):
    """The E-MAML meta-gradient with the exploration stage inside one dataflow launch equals the per-stage launches (and the
    stand-alone exploration launch + promp_reduce_tasks + add of the previous code, reproduced here); the chain is
    deterministic, reports its launch count and leaves its control words zero."""
    torch = _cuda()
    from promp_b200 import _lib
    policy = _policy(M, Do, Da)
    algo = _trpo(policy, M, S1=S1)
    th_l = policy.unpad_flat(policy.theta.cpu().numpy())
    phases = [_fixed_phase(torch, M, N, Do, Da, th_l, 30 + s)[1] for s in range(S1 + 1)]
    for ph in phases:
        ph.adv = torch.randn(M, N, generator=torch.Generator().manual_seed(ph.M + 3)).cuda()
    c = algo.exploration_coeff_dev(phases)

    def run(mode):
        algo.use_chain = mode != 'separate'
        _lib.set_option('chain', 1 if mode == 'dataflow' else 0)
        try:
            res = algo._meta_pass(policy.theta, phases, _lib.OBJ_RATIO, 0.0, [0.0] * S1, want_grad=True, explore=c)
            torch.cuda.synchronize()
        finally:
            _lib.set_option('chain', -1)
        return res['grad'].clone(), res['explore'].clone(), res['stats_all'].clone()
    g_sep, x_sep, st_sep = run('separate')
    g_one, x_one, st_one = run('per_stage')
    g1, x1, st1 = run('dataflow')
    g2, x2, st2 = run('dataflow')
    assert torch.equal(g1, g2) and torch.equal(x1, x2) and torch.equal(st1[..., :3], st2[..., :3])
    assert torch.equal(g_one, g_sep) and torch.equal(x_one, x_sep)          # per-stage launches = stand-alone launches
    assert rel_err(g1.cpu().numpy(), g_sep.cpu().numpy()) < 2e-5
    np.testing.assert_allclose(x1.cpu().numpy(), x_sep.cpu().numpy(), rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(st1[:, :, :3].cpu().numpy(), st_sep[:, :, :3].cpu().numpy(), rtol=2e-5, atol=1e-6)
    # the previous composition: meta-gradient without the term + reduce of the stand-alone exploration gradient + add
    algo.use_chain = False
    base = algo._meta_pass(policy.theta, phases, _lib.OBJ_RATIO, 0.0, [0.0] * S1, want_grad=True)['grad']
    val, gx = algo._exploration_term(policy.theta, phases, True)
    extra = torch.empty_like(base)
    _lib.call('promp_reduce_tasks', M, policy.num_params, _lib.ptr(gx), 1.0 / M, _lib.ptr(extra), _lib.stream())
    assert torch.equal(base + extra, g_sep) and torch.equal(val, x_sep)
    algo.use_chain = True
    ctrl = algo._ws_chain[:4 + 2 * 6 * M].cpu().numpy()
    assert (ctrl == 0).all()
    # launch counts: the stages as the chain sees them (inner grads, outer grad, HVPs, exploration)
    stages = [algo._stage(1 if s > S1 else 0, phases[0], policy.theta, 0, 0) for s in range(2 * S1 + 1)] + \
        [algo._stage(0, phases[0], policy.theta, 0, _lib.OBJ_EXPLORE, adv=c)]
    arr = (_lib.PolicyStage * len(stages))(*stages)
    import ctypes
    nl = getattr(_lib.load(), policy.entries['chain_num_launches'])
    args = (Do, Da, policy.hidden_arg, M, len(stages), ctypes.cast(arr, ctypes.c_void_p))
    for opt, want in ((1, 1), (0, len(stages))):
        _lib.set_option('chain', opt)
        try:
            assert nl(*args) == want
        finally:
            _lib.set_option('chain', -1)


# ------------------------------------------------------------------------------------------------ 5. graph replay
def _trainer(torch, env_name, graph, seed=11, M=4, E=3, H=30):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnvCorner, HalfCheetahRandDirecEnv
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    np.random.seed(seed)
    torch.manual_seed(seed)
    env = normalize(MetaPointEnvCorner(reward_type='dense') if env_name == 'point' else HalfCheetahRandDirecEnv())
    Do, Da = int(np.prod(env.observation_space.shape)), int(np.prod(env.action_space.shape))
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = _trpo(policy, M)
    return Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3, num_inner_grad_steps=1,
                   use_cuda_graph=graph)


def _train(torch, env_name, graph, tmp_path, seed=11):
    from promp_b200.utils import logger
    tr = _trainer(torch, env_name, graph, seed)
    th0 = tr.policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='none')
        tr.train()
        kv = logger.last_dump()
    finally:
        logger.reset()
    assert torch.isfinite(tr.policy.theta).all() and not torch.equal(tr.policy.theta, th0)
    return tr, kv


@pytest.mark.gpu
@pytest.mark.parametrize('env_name', ['cheetah', 'point'])
def test_trainer_replays_emaml_as_graph(env_name, tmp_path):
    """Trainer.train() in 'auto' mode replays TRPOMAML(exploration=True) as one CUDA graph: three iterations, every logged
    scalar finite, the same seed twice bit-identical, the same keys as the eager run.  The eager run's parameters and scalars
    are not compared with the graph run's: the Trainer's two modes draw their action noise from differently keyed Philox
    streams, so their samples differ (the existing ProMP graph-mode tests have the same limit).  Graph against eager on the
    same samples is test_graph_replayed_emaml_step_equals_eager, bit for bit."""
    torch = _cuda()
    tr, kv = _train(torch, env_name, 'auto', tmp_path / 'a')
    assert tr.graph_capturable() and tr._graph_step is not None
    tr2, kv2 = _train(torch, env_name, 'auto', tmp_path / 'b')
    assert torch.equal(tr.policy.theta, tr2.policy.theta)
    for k, v in kv.items():
        if 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert np.isfinite(v), k
            assert v == kv2[k], k
    tr_e, kv_e = _train(torch, env_name, False, tmp_path / 'c')
    assert tr_e._graph_step is None
    assert {k for k in kv if not k.startswith('_')} >= {'LossBefore', 'LossAfter', 'MeanKL', 'MeanKLBefore', 'dLoss'}
    assert set(kv) == set(kv_e)


@pytest.mark.gpu
@pytest.mark.parametrize('env_name', ['cheetah', 'point'])
def test_graph_replayed_emaml_step_equals_eager(env_name):
    """The device part of an E-MAML meta-iteration (optimize_phases: coefficient, CG, line search) captured as a CUDA graph
    and replayed gives the parameters and logged terms of the eager call on the same phases, bit for bit.  (The Trainer's
    eager and graph modes draw their action noise from differently keyed streams, so whole runs are compared per mode.)"""
    torch = _cuda()
    tr = _trainer(torch, env_name, False)
    sampler, proc, algo, policy = tr.sampler, tr.sample_processor, tr.algo, tr.policy
    sampler.update_tasks()
    policy.switch_to_pre_update()
    samples = []
    for step in range(2):
        s = proc.process_samples(sampler.obtain_samples())
        samples.append(s)
        if step == 0:
            algo._adapt(s)
    phases = [s[0].phase for s in samples]
    theta0 = policy.theta.clone()
    algo._adapt_cache = None                    # no launch re-use: the captured pass computes its inner stage the same way
    eager = algo.optimize_phases(phases).clone()
    th_eager = policy.theta.clone()
    for ph in phases:
        ph.invalidate_host()                    # a fresh coefficient, computed inside the capture
    policy.theta.copy_(theta0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        algo.optimize_phases(phases)            # warm-up (allocator pools)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for ph in phases:
        ph.invalidate_host()
    policy.theta.copy_(theta0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = algo.optimize_phases(phases)
    policy.theta.copy_(theta0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager), (out, eager)
    assert torch.equal(policy.theta, th_eager)
    assert float(out[4]) >= 0 or float(out[5]) != 0          # a verdict was reached (accepted step or rejection)
