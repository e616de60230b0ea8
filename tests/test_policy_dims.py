"""Policy kernels for any obs_dim in [1, 19] and action_dim in [1, 8] through the zero-padded parameter layout
(promp_policy_layout and the promp_policy_*_padded entry points).

CPU: the layout table and its bounds.  GPU (-m gpu): forward, adapt, meta-gradients (ProMP, TRPO-MAML incl. the KL
constraint, VPG-MAML with the E-MAML term), variable-length paths, the dataflow chain, determinism and whole Trainer runs
on host envs of new shapes, against the float64 oracle (oracle.tf_half) on the same float32 inputs at the 1e-4 relative
bar; pad entries of every parameter-shaped result must be exactly 0.0; at the shapes of the exact table the padded
entry points must agree with the exact ones.
"""
import math
import pickle

import numpy as np
import pytest

SHAPES = [(1, 1), (3, 1), (5, 3), (8, 2), (11, 3), (19, 8)]
# (obs_dim, action_dim, hidden_sizes, N): N is never a multiple of the 64 / 128-sample tiles
CASES = ([(Do, Da, (64, 64), 333) for Do, Da in SHAPES] + [(Do, Da, (32, 32), 97) for Do, Da in SHAPES]
         + [(5, 3, (16, 16), 97)])
CASE_IDS = ['%dx%d-h%d' % (c[0], c[1], c[2][0]) for c in CASES]


def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_layout_covers_every_supported_shape():
    from promp_b200 import _lib
    lib = _lib.load()
    for hidden in (32, 64):
        for do in range(1, 20):
            for da in range(1, 9):
                oc, ac, hid, P = _lib.policy_layout(do, da, hidden)
                assert oc >= do and ac >= da and hid == hidden
                assert P % 4 == 0 and P == lib.promp_num_params(oc, ac, hidden)


@pytest.mark.parametrize('do,da,hidden', [(0, 2, 64), (20, 2, 64), (5, 9, 64), (5, 3, 48), (5, 0, 32)])
def test_layout_rejects_out_of_range(do, da, hidden):
    from promp_b200 import _lib
    with pytest.raises(_lib.PrompLibraryError, match=r'obs_dim in \[1, 19\], act_dim in \[1, 8\] and hidden 32 or 64'):
        _lib.policy_layout(do, da, hidden)
    assert _lib.load().promp_policy_workspace_bytes_padded(10, 100, do, da, hidden) < 0


def test_padded_chain_workspace_covers_shapes_the_exact_table_rejects():
    import ctypes
    from promp_b200 import _lib
    lib = _lib.load()
    stages = (_lib.PolicyStage * 3)()
    for s, kind in enumerate((0, 0, 1)):
        stages[s].kind, stages[s].N = kind, 500
    ptr = ctypes.cast(stages, ctypes.c_void_p)
    assert lib.promp_policy_chain_workspace_bytes(3, 3, 64, 10, 3, ptr) < 0
    P = _lib.policy_layout(3, 3, 64)[3]
    assert lib.promp_policy_chain_workspace_bytes_padded(3, 3, 64, 10, 3, ptr) >= \
        lib.promp_policy_workspace_bytes_padded(10, 500, 3, 3, 64) > 10 * P * 4


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _policy(M, Do, Da, hidden_sizes, seed=1):
    """A policy with non-trivial logical parameters (log_std and biases included)."""
    from promp_b200.policies import MetaGaussianMLPPolicy
    np.random.seed(seed)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=hidden_sizes)
    th_l = policy.unpad_flat(policy.theta.cpu().numpy()).copy()
    th_l += 0.1 * np.random.RandomState(9).randn(th_l.size).astype(np.float32)
    policy.set_params(th_l)
    return policy


def _logical(policy):
    return policy.unpad_flat(policy.theta.cpu().numpy()).copy()


def _pad_mask(policy):
    mask = np.ones(policy.num_params, dtype=bool)
    mask[policy._pad_index_np] = False
    return mask


def _random_phase(torch, M, N, Do, Da, hidden_sizes, theta_l, seed):
    """Phase data whose old distribution is close to the policy given by the logical parameters theta_l ([P_logical] or
    [M, P_logical])."""
    from promp_b200.samplers.device_data import PhaseData
    from oracle import tf_half as th
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(M, N, Do, generator=g)
    th_t = torch.as_tensor(theta_l)
    th_t = th_t.view(1, -1).expand(M, -1) if th_t.dim() == 1 else th_t
    mean, ls = th.dist_info(th_t, obs, (Do, Da, hidden_sizes))
    old_mean = mean + 0.1 * torch.randn(M, N, Da, generator=g)
    old_ls = (ls + 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
    act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
    adv = torch.randn(M, N, generator=g)
    cpu = dict(obs=obs, act=act, adv=adv, mean=old_mean, log_std=old_ls)
    ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
    ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0])
    ph.adv = adv.cuda()
    return cpu, ph


def _ragged_phase(torch, n_valid, Do, Da, hidden_sizes, theta_l, seed, paths_per_task=3):
    """Variable-length phase: task m has n_valid[m] samples in a few paths; the padding rows hold poison."""
    from promp_b200.samplers.device_data import RaggedPhaseData
    from oracle import tf_half as th
    M = len(n_valid)
    g = torch.Generator().manual_seed(seed)
    lens = []
    for n in n_valid:
        cuts = sorted(set(int(x) for x in torch.randint(1, n, (paths_per_task - 1,), generator=g)))
        edges = [0] + cuts + [n]
        lens.append([b - a for a, b in zip(edges[:-1], edges[1:])])
    ph = RaggedPhaseData(lens, Do, Da, torch.device('cuda'))
    N = ph.N
    obs = torch.randn(M, N, Do, generator=g)
    mean, ls = th.dist_info(torch.as_tensor(theta_l).view(1, -1).expand(M, -1), obs, (Do, Da, hidden_sizes))
    old_mean = mean + 0.1 * torch.randn(M, N, Da, generator=g)
    old_ls = (ls + 0.05 * torch.randn(M, 1, Da, generator=g)).expand(M, N, Da).contiguous()
    act = old_mean + torch.exp(old_ls) * torch.randn(M, N, Da, generator=g)
    adv = torch.randn(M, N, generator=g)
    cpu = []
    for m, n in enumerate(n_valid):
        cpu.append(dict(obs=obs[m:m + 1, :n], act=act[m:m + 1, :n], adv=adv[m:m + 1, :n], mean=old_mean[m:m + 1, :n],
                        log_std=old_ls[m:m + 1, :n]))
        obs[m, n:] = 1e3; act[m, n:] = -50.0; adv[m, n:] = 1e4; old_mean[m, n:] = 7.0
    ph.obs.copy_(obs); ph.act.copy_(act); ph.mean.copy_(old_mean); ph.log_std.copy_(old_ls[:, 0])
    ph.adv = adv.cuda()
    return cpu, ph


def _algo(kind, policy, M, S1=1, **kw):
    from promp_b200.meta_algos import ProMP, TRPOMAML
    if kind == 'promp':
        return ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, learning_rate=1e-3,
                     num_ppo_steps=5, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False, **kw)
    return TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, step_size=0.01, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,hs,N', CASES, ids=CASE_IDS)
def test_forward_matches_oracle(Do, Da, hs, N):
    """get_actions: means and reported log_std for shared (pre-update) and per-task parameters."""
    torch = _cuda()
    from oracle import tf_half as th
    M = 3
    policy = _policy(M, Do, Da, hs)
    assert policy.padded_dims and policy.entries['forward'] == 'promp_policy_forward_padded'
    th_l = _logical(policy)
    obs = np.random.RandomState(3).randn(M, N, Do).astype(np.float32)
    _, infos = policy.get_actions(list(obs))
    mean, ls = th.dist_info(torch.from_numpy(th_l).view(1, -1).expand(M, -1).double(), torch.from_numpy(obs).double(),
                            (Do, Da, hs))
    got = np.stack([np.stack([i['mean'] for i in task]) for task in infos])
    assert got.shape == (M, N, Da)
    assert rel_err(got, mean.numpy()) < 1e-5
    np.testing.assert_array_equal(np.stack([task[0]['log_std'] for task in infos]),
                                  np.maximum(np.float32(ls[:, 0].numpy()), np.float32(policy.min_log_std)))
    # per-task parameters (post-update sampling): stride P
    tasks_l = th_l[None] + 0.05 * np.random.RandomState(4).randn(M, th_l.size).astype(np.float32)
    policy.update_task_parameters(torch.from_numpy(policy.pad_flat(tasks_l)).cuda())
    _, infos = policy.get_actions(list(obs))
    mean, ls = th.dist_info(torch.from_numpy(tasks_l).double(), torch.from_numpy(obs).double(), (Do, Da, hs))
    got = np.stack([np.stack([i['mean'] for i in task]) for task in infos])
    assert rel_err(got, mean.numpy()) < 1e-5
    np.testing.assert_array_equal(np.stack([task[0]['log_std'] for task in infos]), np.float32(ls[:, 0].numpy()))


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,hs,N', CASES, ids=CASE_IDS)
@pytest.mark.parametrize('inner', ['likelihood_ratio', 'log_likelihood'])
def test_adapt_matches_oracle(Do, Da, hs, N, inner):
    """MAMLAlgo._adapt pre-update (shared theta), then per-task, against th.adapt; pads of theta' stay exactly zero."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.samplers.device_data import SamplesData
    M = 5
    policy = _policy(M, Do, Da, hs)
    algo = _algo('trpo', policy, M, inner_type=inner)
    dims, th_l = (Do, Da, hs), _logical(policy)
    cpu, ph = _random_phase(torch, M, N, Do, Da, hs, th_l, 1)
    samples = [SamplesData(ph, m) for m in range(M)]
    policy.switch_to_pre_update()
    algo._adapt(samples)
    want = th.adapt(torch.from_numpy(th_l).view(1, -1).expand(M, -1).contiguous(), cpu, dims, 0.1, inner)
    got = policy.theta_tasks.cpu().numpy()
    mask = _pad_mask(policy)
    assert np.all(got[:, mask] == 0.0) and np.all(algo.last_inner_grad.cpu().numpy()[:, mask] == 0.0)
    g_want = (torch.from_numpy(th_l).view(1, -1) - want) / 0.1
    assert rel_err(policy.unpad_flat(algo.last_inner_grad.cpu().numpy()), g_want.numpy()) < 1e-4
    np.testing.assert_allclose(policy.unpad_flat(got), want.numpy(), rtol=1e-5, atol=2e-6)
    algo._adapt(samples)
    want2 = th.adapt(want, cpu, dims, 0.1, inner)
    got2 = policy.theta_tasks.cpu().numpy()
    assert np.all(got2[:, mask] == 0.0)
    np.testing.assert_allclose(policy.unpad_flat(got2), want2.numpy(), rtol=1e-5, atol=4e-6)


def _check_meta_gradient(torch, kind, policy, algo, phases, cpus, dims, S1):
    """ProMP: _objective_pass gradient and loss terms; TRPO: loss / KL values, loss gradient and KL-constraint gradient."""
    from oracle import tf_half as th
    th_l = _logical(policy)
    t64 = torch.tensor(th_l, dtype=torch.float64, requires_grad=True)
    coeff = list(algo.inner_kl_coeff) if kind == 'promp' else None
    obj, ikl, okl = th.meta_objective(t64, cpus, dims, 0.1, kind, 0.3, coeff)
    (g_want,) = torch.autograd.grad(obj, t64)
    mask = _pad_mask(policy)
    if kind == 'promp':
        res = algo._objective_pass(phases, want_grad=True)
        terms = algo.loss_terms(res).cpu().numpy()
        assert abs(terms[0] - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
        np.testing.assert_allclose(terms[1:1 + S1], ikl.detach().numpy(), rtol=1e-3, atol=1e-6)
        np.testing.assert_allclose(terms[1 + S1], float(okl), rtol=1e-3, atol=1e-6)
        g_got = res['grad'].cpu().numpy()
    else:
        g_got = np.asarray(algo.eval_gradient(policy.theta, phases, 'loss'))
        loss, klv = algo.eval_scalars(policy.theta, phases)
        assert abs(loss - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
        assert abs(klv - float(okl)) < 1e-3 * max(1e-3, abs(float(okl)))
        (gk_want,) = torch.autograd.grad(th.meta_objective(t64, cpus, dims, 0.1, kind)[2], t64)
        gk_got = np.asarray(algo.eval_gradient(policy.theta, phases, 'kl'))
        assert np.all(gk_got[mask] == 0.0)
        assert rel_err(policy.unpad_flat(gk_got), gk_want.numpy()) < 1e-4
    assert np.all(g_got[mask] == 0.0)
    err = rel_err(policy.unpad_flat(g_got), g_want.numpy())
    assert err < 1e-4, err


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,hs,N', CASES, ids=CASE_IDS)
@pytest.mark.parametrize('S1', [1, 2])
@pytest.mark.parametrize('kind', ['promp', 'trpo'])
def test_meta_gradient_matches_oracle(Do, Da, hs, N, S1, kind):
    torch = _cuda()
    M = 4
    N = N if S1 == 1 else 150
    policy = _policy(M, Do, Da, hs)
    algo = _algo(kind, policy, M, S1=S1)
    th_l = _logical(policy)
    cpus, phases = [], []
    for s in range(S1 + 1):
        c, p = _random_phase(torch, M, N, Do, Da, hs, th_l, 10 + s)
        cpus.append({k: v.double() for k, v in c.items()})
        phases.append(p)
    _check_meta_gradient(torch, kind, policy, algo, phases, cpus, (Do, Da, hs), S1)


@pytest.mark.gpu
@pytest.mark.parametrize('tc', [0, 1])
@pytest.mark.parametrize('kind', ['promp', 'trpo'])
def test_ragged_adapt_and_meta_gradient_match_oracle(kind, tc):
    """Variable-length paths (n_valid): the adapt step per task on its trimmed data, and the meta-gradient."""
    torch = _cuda()
    from promp_b200 import _lib
    from oracle import tf_half as th
    M, Do, Da, hs = 5, 11, 3, (64, 64)
    dims = (Do, Da, hs)
    policy = _policy(M, Do, Da, hs)
    algo = _algo(kind, policy, M)
    th_l = _logical(policy)
    nv = [[130, 517, 64, 1000, 333], [257, 90, 700, 128, 411]]
    cpus, phases = [], []
    for s in range(2):
        c, p = _ragged_phase(torch, nv[s], Do, Da, hs, th_l, 20 + s)
        cpus.append(c); phases.append(p)
    mask = _pad_mask(policy)
    try:
        _lib.set_option('tensor_cores', tc)
        policy.switch_to_pre_update()
        algo._adapt_launch(phases[0])
        got = policy.theta_tasks.cpu().numpy()
        assert np.all(got[:, mask] == 0.0)
        for m in range(M):
            want = th.adapt(torch.from_numpy(th_l).view(1, -1), cpus[0][m], dims, 0.1)
            np.testing.assert_allclose(policy.unpad_flat(got[m]), want[0].numpy(), rtol=1e-5, atol=2e-6)
        policy.switch_to_pre_update()
        coeff = list(algo.inner_kl_coeff) if kind == 'promp' else None
        g_want, obj_want, okl_want = 0.0, 0.0, 0.0
        for m in range(M):
            t64 = torch.tensor(th_l, dtype=torch.float64, requires_grad=True)
            data_m = [{k: v.double() for k, v in cpus[s][m].items()} for s in range(2)]
            obj, _, okl = th.meta_objective(t64, data_m, dims, 0.1, kind, 0.3, coeff)
            (gm,) = torch.autograd.grad(obj, t64)
            g_want = g_want + gm.numpy() / M
            obj_want += float(obj) / M
            okl_want += float(okl) / M
        if kind == 'promp':
            res = algo._objective_pass(phases, want_grad=True)
            loss = float(algo.loss_terms(res).cpu().numpy()[0])
            g_got = res['grad'].cpu().numpy()
        else:
            g_got = np.asarray(algo.eval_gradient(policy.theta, phases, 'loss'))
            loss, klv = algo.eval_scalars(policy.theta, phases)
            assert abs(klv - okl_want) < 1e-3 * max(1e-3, abs(okl_want))
    finally:
        _lib.set_option('tensor_cores', 1)
    assert abs(loss - obj_want) < 1e-4 * max(1.0, abs(obj_want))
    assert np.all(g_got[mask] == 0.0)
    assert rel_err(policy.unpad_flat(g_got), g_want) < 1e-4


@pytest.mark.gpu
def test_vpg_maml_with_exploration_term_matches_oracle():
    """VPGMAML(exploration=True) (E-MAML term, fixed-horizon paths) on a new shape: gradient, loss and the Adam step."""
    torch = _cuda()
    from oracle import tf_half as th
    from promp_b200.meta_algos import VPGMAML
    from promp_b200.samplers.device_data import SamplesData
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    M, N, Do, Da, hs = 4, 180, 5, 3, (64, 64)
    np.random.seed(4)
    from promp_b200.policies import MetaGaussianMLPPolicy
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=hs)
    algo = VPGMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                   inner_type='log_likelihood', exploration=True)
    dims, th_l = (Do, Da, hs), _logical(policy)
    cpus, phases = [], []
    for s in range(2):
        c, p = _random_phase(torch, M, N, Do, Da, hs, th_l, 110 + s)
        rew = torch.randn(M, N, generator=torch.Generator().manual_seed(5 + s)) + torch.arange(M).view(-1, 1).float()
        p.rew.copy_(rew)
        keep = p.adv.clone()
        run_process_kernel(p, 0.99, 1.0, 1e-5, 1, True, False)
        p.adv = keep
        c = {k: v.double() for k, v in c.items()}
        r64 = rew.double()
        c['adj_avg_rewards'] = (r64 - r64.mean()) / (r64.std(unbiased=False) + 1e-8)
        cpus.append(c); phases.append(p)
    t64 = torch.tensor(th_l, dtype=torch.float64, requires_grad=True)
    obj, _, _ = th.meta_objective(t64, cpus, dims, 0.1, 'vpg', inner_type='log_likelihood', exploration=True)
    (g_want,) = torch.autograd.grad(obj, t64)
    res = algo._objective_pass(phases, want_grad=True)
    g_got = res['grad'].cpu().numpy()
    mask = _pad_mask(policy)
    assert np.all(g_got[mask] == 0.0)
    assert rel_err(policy.unpad_flat(g_got), g_want.numpy()) < 1e-4
    assert abs(float(algo.loss_terms(res)[0]) - float(obj)) < 1e-4 * max(1.0, abs(float(obj)))
    algo.optimize_policy([[SamplesData(p, m) for m in range(M)] for p in phases], log=False)
    want = th.TF1Adam(th_l.size).step(torch.tensor(th_l), g_want.float())
    assert np.all(policy.theta.cpu().numpy()[mask] == 0.0)
    np.testing.assert_allclose(_logical(policy), want.numpy(), rtol=0, atol=2e-5)


@pytest.mark.gpu
def test_pad_entries_stay_exactly_zero_through_training_steps():
    """Gradient of _objective_pass, theta and both Adam slots after ProMP.optimize_policy (5 epochs), theta and theta_tasks
    after a TRPOMAML step: every pad entry is exactly 0.0."""
    torch = _cuda()
    from promp_b200.samplers.device_data import SamplesData
    M, N, Do, Da, hs = 4, 333, 5, 3, (64, 64)
    mask = None
    for kind in ('promp', 'trpo'):
        policy = _policy(M, Do, Da, hs)
        algo = _algo(kind, policy, M)
        mask = _pad_mask(policy)
        th_l = _logical(policy)
        phases = [_random_phase(torch, M, N, Do, Da, hs, th_l, 30 + s)[1] for s in range(2)]
        samples = [[SamplesData(p, m) for m in range(M)] for p in phases]
        policy.switch_to_pre_update()
        algo._adapt(samples[0])
        assert np.all(policy.theta_tasks.cpu().numpy()[:, mask] == 0.0)
        policy.switch_to_pre_update()
        if kind == 'promp':
            res = algo._objective_pass(phases, want_grad=True)
            assert np.all(res['grad'].cpu().numpy()[mask] == 0.0)
        algo.optimize_policy(samples, log=False)
        theta = policy.theta.cpu().numpy()
        assert np.all(theta[mask] == 0.0)
        if kind == 'promp':
            assert not np.array_equal(policy.unpad_flat(theta), th_l)
            assert np.all(algo.optimizer.m.cpu().numpy()[mask] == 0.0) and np.all(algo.optimizer.v.cpu().numpy()[mask] == 0.0)
            assert np.any(algo.optimizer.v.cpu().numpy() != 0.0)
        else:
            algo._adapt(samples[0])
            assert np.all(policy.theta_tasks.cpu().numpy()[:, mask] == 0.0)


def _exact_to_padded_index(Do, Da, hidden):
    """Positions of the exact layout's parameters inside the padded layout of the same logical shape."""
    from promp_b200 import _lib
    oc, ac, _, P = _lib.policy_layout(Do, Da, hidden)
    idx, off = [], 0
    for shape, cap in zip(((Do, hidden), (hidden,), (hidden, hidden), (hidden,), (hidden, Da), (Da,), (1, Da)),
                          ((oc, hidden), (hidden,), (hidden, hidden), (hidden,), (hidden, ac), (ac,), (1, ac))):
        grid = np.arange(int(np.prod(cap))).reshape(cap) + off
        idx.append(grid[tuple(slice(0, n) for n in shape)].reshape(-1))
        off += int(np.prod(cap))
    return np.concatenate(idx), P


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da', [(2, 2), (4, 2), (17, 6)])
@pytest.mark.parametrize('hidden', [64, 32])
def test_padded_entries_match_exact_ones(Do, Da, hidden):
    """At the shapes of the exact table the *_padded entry points (bucket kernels), unpadded, give the exact kernels'
    gradient, HVP and forward to 1e-6 relative (different tile mappings sum in different orders)."""
    torch = _cuda()
    from promp_b200 import _lib
    M, N = 6, 333
    hs = (hidden, hidden)
    policy = _policy(M, Do, Da, hs)
    assert not policy.padded_dims
    algo = _algo('promp', policy, M)
    idx, P_pad = _exact_to_padded_index(Do, Da, hidden)
    P = policy.num_params
    _, ph = _random_phase(torch, M, N, Do, Da, hs, _logical(policy), 7)
    theta_pad = torch.zeros(P_pad, device='cuda')
    theta_pad[torch.from_numpy(idx).cuda()] = policy.theta
    vec = torch.randn(M, P, generator=torch.Generator().manual_seed(3)).cuda()
    vec_pad = torch.zeros(M, P_pad, device='cuda')
    vec_pad[:, torch.from_numpy(idx).cuda()] = vec
    obs = ph.obs.contiguous()

    def run(params, Pn, v):
        g = torch.empty(M, Pn, device='cuda')
        newp = torch.empty(M, Pn, device='cuda')
        hv = torch.empty(M, Pn, device='cuda')
        st = torch.empty(M, 4, device='cuda')
        algo._grad(ph, params, 0, _lib.OBJ_RATIO, kl_coeff=0.01, clip_log_std=1, grad=g, out_params=newp, sgd_lr=0.1, stats=st)
        algo._hvp(ph, newp, Pn, v, hv, 5e-4, 0)
        mean = torch.empty(M, N, Da, device='cuda')
        _lib.call(policy.entries['forward'], Do, Da, hidden, M, N, _lib.ptr(newp), Pn, _lib.ptr(obs), _lib.ptr(mean), _lib.stream())
        torch.cuda.synchronize()
        return g, hv, mean, st
    exact = run(policy.theta, P, vec)
    policy.entries = {k: v.replace('promp_policy_' + k, 'promp_policy_' + k + '_padded') for k, v in policy.entries.items()}
    padded = run(theta_pad, P_pad, vec_pad)
    sel = torch.from_numpy(idx).cuda()
    pairs = dict(grad=(padded[0][:, sel], exact[0]), hvp=(padded[1][:, sel], exact[1]), mean=(padded[2], exact[2]),
                 stats=(padded[3][:, :3], exact[3][:, :3]))
    for name, (a, b) in pairs.items():
        e = rel_err(a.cpu().numpy(), b.cpu().numpy())
        print('padded vs exact %dx%d h%d %s: rel err %.3g, bitwise equal %s' % (Do, Da, hidden, name, e, bool(torch.equal(a, b))))
        assert e <= 1e-6, (name, e)
    pad = np.ones(P_pad, dtype=bool)
    pad[idx] = False
    assert np.all(padded[0].cpu().numpy()[:, pad] == 0.0) and np.all(padded[1].cpu().numpy()[:, pad] == 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,M,N,S1', [(11, 3, 10, 700, 1), (19, 8, 5, 391, 2), (1, 1, 40, 2000, 1)])
def test_padded_chain_matches_separate_launches(Do, Da, M, N, S1):
    """promp_policy_chain_padded (one dataflow launch) against the same stages as separate padded launches; the chain is
    bitwise deterministic and leaves its control words zero; num_launches reports what runs."""
    torch = _cuda()
    import ctypes
    from promp_b200 import _lib
    policy = _policy(M, Do, Da, (64, 64))
    algo = _algo('promp', policy, M, S1=S1)
    th_l = _logical(policy)
    phases = [_random_phase(torch, M, N, Do, Da, (64, 64), th_l, 20 + s)[1] for s in range(S1 + 1)]
    stages = (_lib.PolicyStage * (2 * S1 + 1))()
    for s in range(2 * S1 + 1):
        stages[s].kind, stages[s].N = (0 if s <= S1 else 1), N
    sp = ctypes.cast(stages, ctypes.c_void_p)
    lib = _lib.load()

    def run(chain, want_grad=True):
        algo.use_chain = chain
        _lib.set_option('chain', 1)
        try:
            assert getattr(lib, policy.entries['chain_num_launches'])(Do, Da, 64, M, 2 * S1 + 1, sp) == 1
            res = algo._objective_pass(phases, want_grad=want_grad, reduce=False)
            torch.cuda.synchronize()
        finally:
            _lib.set_option('chain', -1)
        return (res['grad_tasks'].clone() if want_grad else None), res['stats_all'].clone()
    g_ref, st_ref = run(False)
    g1, st1 = run(True)
    g2, st2 = run(True)
    assert torch.equal(g1, g2) and torch.equal(st1, st2)
    mask = _pad_mask(policy)
    assert np.all(g1.cpu().numpy()[:, mask] == 0.0)
    for m in range(M):
        assert rel_err(g1[m].cpu().numpy(), g_ref[m].cpu().numpy()) < 2e-5
    np.testing.assert_allclose(st1[:, :, :3].cpu().numpy(), st_ref[:, :, :3].cpu().numpy(), rtol=2e-5, atol=1e-6)
    _, st3 = run(True, want_grad=False)
    np.testing.assert_allclose(st3[:, :, :3].cpu().numpy(), st_ref[:, :, :3].cpu().numpy(), rtol=2e-5, atol=1e-6)
    ctrl = algo._ws_chain[:4 + 2 * 6 * M].cpu().numpy()
    assert (ctrl == 0).all()
    _lib.set_option('chain', 0)
    try:
        assert getattr(lib, policy.entries['chain_num_launches'])(Do, Da, 64, M, 2 * S1 + 1, sp) == 2 * S1 + 1
    finally:
        _lib.set_option('chain', -1)


@pytest.mark.gpu
@pytest.mark.parametrize('hs', [(64, 64), (32, 32)])
def test_padded_launches_are_deterministic(hs):
    torch = _cuda()
    M, N, Do, Da = 7, 1000, 11, 3
    policy = _policy(M, Do, Da, hs)
    algo = _algo('promp', policy, M)
    th_l = _logical(policy)
    phases = [_random_phase(torch, M, N, Do, Da, hs, th_l, 40 + s)[1] for s in range(2)]
    outs = []
    for _ in range(2):
        algo.use_chain = False
        a = algo._objective_pass(phases, want_grad=True, reduce=False)
        algo.use_chain = True
        b = algo._objective_pass(phases, want_grad=True, reduce=False)
        outs.append((a['grad_tasks'].clone(), a['stats_all'][..., :3].clone(), b['grad_tasks'].clone(), b['stats_all'][..., :3].clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


# ---- end to end on host envs of new shapes ---------------------------------------------------------------------------------
class IntegratorEnv(object):
    """The reference's 1-d integrator test env (tests/test_samplers.py:13-55): state += goal - action, obs = 100 * state +
    goal, reward = goal - action.  obs_dim 1, action_dim 1, fixed-horizon paths."""

    def __init__(self):
        self.state, self.goal = np.zeros(1), 0

    def sample_tasks(self, n_tasks):
        return np.random.choice(100, n_tasks, replace=False)

    def set_task(self, task):
        self.goal = task

    def get_task(self):
        return self.goal

    def step(self, action):
        self.state += self.goal - action
        return self.state * 100 + self.goal, (self.goal - action)[0], 0, {}

    def reset(self):
        self.state = np.zeros(1)
        return self.state

    def log_diagnostics(self, paths, prefix=''):
        pass


class ReachEnv(object):
    """A linear 5-d reaching task driven by a 3-d action: s' = s + 0.2 * B a, reward = -|s' - goal|; a path ends early
    once |s' - goal| < 0.4 or after a step budget drawn at reset (3..9 steps), so paths have different lengths.
    obs = s - goal."""
    B = np.random.RandomState(0).randn(5, 3) / np.sqrt(3)

    def __init__(self):
        self.s, self.goal = np.zeros(5), np.zeros(5)

    def sample_tasks(self, n_tasks):
        return [0.5 * np.random.randn(5) for _ in range(n_tasks)]

    def set_task(self, task):
        self.goal = np.asarray(task, dtype=np.float64)

    def get_task(self):
        return self.goal

    def step(self, action):
        self.s = self.s + 0.2 * self.B.dot(np.clip(np.asarray(action, dtype=np.float64), -1, 1))
        dist = float(np.linalg.norm(self.s - self.goal))
        self.t += 1
        return self.s - self.goal, -dist, dist < 0.4 or self.t >= self.budget, {}

    def reset(self):
        self.s = 0.1 * np.random.randn(5)
        self.t, self.budget = 0, np.random.randint(3, 10)
        return self.s - self.goal

    def log_diagnostics(self, paths, prefix=''):
        pass


@pytest.mark.gpu
@pytest.mark.parametrize('env_cls', [IntegratorEnv, ReachEnv])
@pytest.mark.parametrize('algo_name', ['promp', 'trpo', 'vpg'])
def test_trainer_runs_on_host_envs_of_new_shapes(env_cls, algo_name, tmp_path):
    torch = _cuda()
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP, TRPOMAML, VPGMAML
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.utils import logger
    M, E, H = 4, 3, 12
    np.random.seed(11)
    env = env_cls()
    Do, Da = (1, 1) if env_cls is IntegratorEnv else (5, 3)
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64))
    assert policy.padded_dims
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    if algo_name == 'promp':
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=3, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=True)
    elif algo_name == 'trpo':
        algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, step_size=0.01)
    else:
        algo = VPGMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3)
    theta0 = policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='none')
        Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                num_inner_grad_steps=1).train()
        kv = logger.last_dump()
    finally:
        logger.reset()
    assert kv['Itr'] == 2
    for key in ('Step_0-AverageReturn', 'Step_1-AverageReturn', 'Step_0-AveragePolicyStd', 'Step_1-AveragePolicyStd',
                'Step_1-NumTrajs', 'LossBefore', 'LossAfter'):
        assert key in kv and np.isfinite(kv[key]), key
    assert all(np.isfinite(v) for v in kv.values() if isinstance(v, (float, int, np.floating)))
    if env_cls is ReachEnv:
        assert kv['Step_0-NumTrajs'] > M * E          # early termination: more, shorter paths than envs
    theta = policy.theta.cpu().numpy()
    assert np.all(theta[_pad_mask(policy)] == 0.0) and not torch.equal(policy.theta, theta0)
    # pickling stores the logical parameters; the round trip reproduces the policy's means bitwise
    policy.switch_to_pre_update()
    state = policy.__getstate__()
    assert state['network_params']['mean_network/hidden_0/kernel'].shape == (Do, 64)
    assert state['network_params']['log_std_network/log_std_var'].shape == (1, Da)
    clone = pickle.loads(pickle.dumps(policy))
    obs = list(np.random.RandomState(5).randn(M, 9, Do).astype(np.float32))
    _, infos = policy.get_actions(obs)
    _, infos2 = clone.get_actions(obs)
    for a, b in zip(sum(infos, []), sum(infos2, [])):
        np.testing.assert_array_equal(a['mean'], b['mean'])
        np.testing.assert_array_equal(a['log_std'], b['log_std'])


@pytest.mark.gpu
def test_out_of_range_shapes_raise_at_construction():
    _cuda()
    from promp_b200.policies import MetaGaussianMLPPolicy
    for Do, Da in ((20, 2), (0, 2), (5, 9)):
        with pytest.raises(NotImplementedError, match=r'obs_dim in \[1, 19\] and action_dim in \[1, 8\]'):
            MetaGaussianMLPPolicy(name="p", obs_dim=Do, action_dim=Da, meta_batch_size=2)
