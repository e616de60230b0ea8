"""Trainable per-parameter inner step sizes (Meta-SGD, `trainable_inner_step_size=True`, ref meta_algos/base.py:98, 210,
303-313): theta_{s+1} = theta_s - alpha * g_s with alpha [P] trained by the outer Adam together with theta.

CPU tests check the host logic: the stage lists carry alpha on the inner gradient and HVP stages, the reference-shaped
`step_sizes` dict, the TRPO-MAML rejection.  GPU tests check the theta- and alpha-gradients against float64 autograd through
oracle/tf_half.meta_objective (whose inner step broadcasts a [P] step-size tensor), the scalar path at alpha = inner_lr, one
Adam step over [theta; alpha], CUDA-graph replay and snapshot / restore."""
import os

import numpy as np
import pytest
import torch

import test_policy_oracle as po
from oracle import tf_half as th


def _cpu_policy(M, monkeypatch, Do=2, Da=2, hidden=64):
    from promp_b200 import _lib
    from promp_b200.policies import MetaGaussianMLPPolicy
    monkeypatch.setattr(_lib, 'require_cuda', lambda: _lib.load())
    return MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(hidden, hidden),
                                 device='cpu')


def test_trpo_maml_rejects_trainable_step_size(monkeypatch):
    from promp_b200.meta_algos import TRPOMAML
    pol = _cpu_policy(2, monkeypatch)
    with pytest.raises(NotImplementedError, match='trainable_inner_step_size'):
        TRPOMAML(policy=pol, inner_lr=0.1, meta_batch_size=2, num_inner_grad_steps=1, trainable_inner_step_size=True)
    with pytest.raises(NotImplementedError):
        TRPOMAML(pol, 0.1, 2, 1, True)


@pytest.mark.parametrize('Do,Da', [(2, 2), (3, 1)])
def test_step_sizes_dict_has_the_reference_keys_and_shapes(Do, Da, monkeypatch):
    from promp_b200.meta_algos import ProMP, VPGMAML
    pol = _cpu_policy(2, monkeypatch, Do, Da)
    for cls in (ProMP, VPGMAML):
        algo = cls(policy=pol, inner_lr=0.05, meta_batch_size=2, num_inner_grad_steps=1, trainable_inner_step_size=True)
        assert algo.alpha.shape == (pol.num_params,) and bool((algo.alpha == np.float32(0.05)).all())
        assert algo.optimizer.m_alpha.shape == (pol.num_params,) and algo.optimizer.last_grad_full.shape == (2 * pol.num_params,)
        d = algo.step_sizes
        assert list(d) == list(pol.param_shapes)
        for k, shape in pol.param_shapes.items():
            assert d[k].shape == shape and np.all(d[k] == np.float32(0.05))
    fixed = ProMP(policy=pol, inner_lr=0.05, meta_batch_size=2, num_inner_grad_steps=1)
    assert fixed.alpha is None and fixed.optimizer.m_alpha is None
    assert all(np.all(v == np.float32(0.05)) for v in fixed.step_sizes.values())


@pytest.mark.parametrize('algo_kind,S1', [('promp', 1), ('promp', 3), ('vpg', 2)])
def test_stage_lists_carry_the_step_sizes(algo_kind, S1, monkeypatch):
    """Host side only (launches recorded, none run): every inner gradient stage with out_params and every HVP stage points at
    alpha, HVP stages get inner_lr = 1, the outer stage does not; the (v_{s+1}, g_s) pairs are the HVP inputs and the inner
    gradients in step order; _adapt goes through the stage path without launch re-use."""
    from promp_b200 import _lib
    from promp_b200.meta_algos import ProMP, VPGMAML
    from promp_b200.samplers.device_data import PhaseData
    M, N = 3, 200
    pol = _cpu_policy(M, monkeypatch)
    if algo_kind == 'promp':
        algo = ProMP(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, num_ppo_steps=1,
                     trainable_inner_step_size=True)
    else:
        algo = VPGMAML(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, trainable_inner_step_size=True)
    calls = []

    def record(name, *args):
        if name in ('promp_policy_chain', 'promp_policy_chain_padded'):
            n, arr = args[5], args[6]
            st = (_lib.PolicyStage * n).from_address(arr.value)
            calls.append(dict(name=name, stages=[(s.kind, s.out_params, s.grad, s.vec, s.step_size, s.inner_lr) for s in st],
                              skip=(args[7], args[8])))
        else:
            calls.append(dict(name=name, args=args))
    monkeypatch.setattr(_lib, 'call', record)
    monkeypatch.setattr(_lib, 'ptr', lambda t: None if t is None else t.data_ptr())
    monkeypatch.setattr(_lib, 'stream', lambda: None)
    phases = []
    for s in range(S1 + 1):
        ph = PhaseData(M, 1, N, 2, 2, torch.device('cpu'))
        ph.adv = torch.zeros(M, N)
        phases.append(ph)
    alpha = algo.alpha.data_ptr()
    algo.adapt_phase(phases[0])
    assert algo._adapt_cache is None
    assert len(calls) == 1 and calls[0]['stages'][0][4] == alpha and calls[0]['skip'] == (None, None)
    calls.clear()
    res = algo._objective_pass(phases, want_grad=True, **({'reduce': False} if algo_kind == 'promp' else {}))
    stages = [s for c in calls if 'stages' in c for s in c['stages']]
    assert [s[0] for s in stages] == [0] * (S1 + 1) + [1] * S1
    for s in stages[:S1]:
        assert s[4] == alpha
    assert stages[S1][4] is None and stages[S1][1] is None
    for s in stages[S1 + 1:]:
        assert s[4] == alpha and s[5] == 1.0
    pairs = res['sgd_pairs']
    assert len(pairs) == S1
    for s in range(S1):
        hvp = stages[S1 + 1 + (S1 - 1 - s)]                 # HVP stages run s = S1-1 .. 0
        assert pairs[s][0].data_ptr() == hvp[3] and pairs[s][1].data_ptr() == stages[s][2]
    if algo_kind == 'vpg':
        assert res['grad'].shape == (2 * pol.num_params,)
        assert any(c['name'] == 'promp_reduce_tasks_sgd' and c['args'][2] is None for c in calls)


@pytest.mark.parametrize('name', ['promp_small', 'promp_s3', 'vpg_small'])
def test_oracle_matches_reference_graph_with_trainable_step_sizes(golden_dir, name):
    """The float64 oracle with a [P] step-size tensor (theta - alpha * g) == the unmodified reference graph with
    trainable_inner_step_size=True at a non-uniform alpha (tests/golden/tf_half_meta_sgd.npz, tools/make_meta_sgd_golden.py):
    the objective and its gradients with respect to the policy variables and the step-size variables."""
    from oracle import tf_cases
    from test_relu_policy import _oracle_data
    G = np.load(os.path.join(golden_dir, 'tf_half_meta_sgd.npz'))
    case = tf_cases.make_case(name)
    pre = name + '/f64/'
    dims = (case['Do'], case['Da'], (case['hidden'],) * 2)
    data = _oracle_data(case, torch.float64)
    t = torch.tensor(case['theta'], dtype=torch.float64, requires_grad=True)
    a = torch.tensor(G[pre + 'alpha'], dtype=torch.float64, requires_grad=True)
    obj, _, _ = th.meta_objective(t, data, dims, a, case['algo'], 0.3, [5e-4] * (case['S'] - 1),
                                  case.get('inner_type', 'likelihood_ratio'))
    gt, ga = torch.autograd.grad(obj, (t, a))
    rel = lambda x, y: float(np.linalg.norm(x - y) / np.linalg.norm(y))
    assert abs(float(obj.detach()) - float(G[pre + 'loss'])) <= 1e-9 + 1e-6 * abs(float(G[pre + 'loss']))
    assert rel(gt.numpy(), G[pre + 'grad']) < 1e-6
    assert rel(ga.numpy(), G[pre + 'grad_alpha']) < 1e-6
    # and alpha matters: the uniform step size gives another alpha-gradient
    a0 = torch.full_like(a, float(np.float32(0.1))).requires_grad_(True)
    (ga0,) = torch.autograd.grad(th.meta_objective(t, data, dims, a0, case['algo'], 0.3, [5e-4] * (case['S'] - 1),
                                                   case.get('inner_type', 'likelihood_ratio'))[0], a0)
    assert rel(ga0.numpy(), G[pre + 'grad_alpha']) > 1e-3


# ------------------------------------------------------------------------------------------------------------- GPU
class Case(object):
    def __init__(self, cid, algo, S1, Do, Da, hidden, M=4, N=300, n_valid=None, chain=-1, explore=False):
        self.cid, self.algo, self.S1, self.Do, self.Da, self.hidden = cid, algo, S1, Do, Da, hidden
        self.M, self.N, self.n_valid, self.chain, self.explore = M, N, n_valid, chain, explore


CASES = [
    Case('promp-s1-point-h64', 'promp', 1, 2, 2, 64),
    Case('promp-s2-cheetah-h64-dataflow', 'promp', 2, 17, 6, 64, M=20, N=1000, chain=1),
    Case('promp-s2-cheetah-h64-perstage', 'promp', 2, 17, 6, 64, chain=0),
    Case('promp-s3-point-h64-dataflow', 'promp', 3, 2, 2, 64, M=20, N=1000, chain=1),
    Case('promp-s3-point-h32', 'promp', 3, 2, 2, 32),
    Case('promp-s1-padded-h64', 'promp', 1, 3, 1, 64),
    Case('promp-s2-point-h64-ragged', 'promp', 2, 2, 2, 64, n_valid=[[300, 250, 131, 200], [280, 300, 90, 17], [1, 300, 150, 299]]),
    Case('vpg-s1-cheetah-h32', 'vpg', 1, 17, 6, 32),
    Case('vpg-s2-point-h64-explore', 'vpg', 2, 2, 2, 64, explore=True),
]


class Setup(object):
    def __init__(self, c, alpha_scale=0.5):
        from promp_b200.meta_algos import ProMP, VPGMAML
        from promp_b200.policies import MetaGaussianMLPPolicy
        from promp_b200.samplers.device_data import PhaseData, RaggedPhaseData
        self.c = c
        rng = np.random.RandomState(9000 + sum(map(ord, c.cid)))
        M, Do, Da, H = c.M, c.Do, c.Da, c.hidden
        self.dims = (Do, Da, (H, H))
        self.pol = pol = MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(H, H))
        theta = th.init_params(*self.dims, rng=rng).astype(np.float64) + 0.1 * rng.randn(th.num_params(*self.dims))
        theta[-Da:] = rng.uniform(-0.7, 0.0, size=Da)
        self.theta = theta.astype(np.float32)
        pol.set_params(self.theta)
        kw = dict(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=c.S1, trainable_inner_step_size=True)
        if c.algo == 'promp':
            self.algo = ProMP(num_ppo_steps=1, clip_eps=po.CLIP_EPS, init_inner_kl_penalty=5e-3, adaptive_inner_kl_penalty=False,
                              **kw)
        else:
            self.algo = VPGMAML(exploration=c.explore, **kw)
        # a non-uniform alpha: inner_lr * exp(U(-1/2, 1/2)), in the device layout
        self.alpha = (0.1 * np.exp(rng.uniform(-alpha_scale, alpha_scale, th.num_params(*self.dims)))).astype(np.float32)
        self.algo.alpha.copy_(torch.from_numpy(pol.pad_flat(self.alpha)))
        self.phases, self.cpus = [], []
        t64 = torch.from_numpy(self.theta).double().view(1, -1).expand(M, -1)
        for s in range(c.S1 + 1):
            nv = c.n_valid[s] if c.n_valid is not None else None
            N = c.N
            obs = rng.randn(M, N, Do)
            with torch.no_grad():
                mean, ls = th.dist_info(t64, torch.from_numpy(obs), self.dims, pol.min_log_std)
            old_mean = mean.numpy() + 0.1 * rng.randn(M, N, Da)
            old_ls = ls.numpy() + 0.05 * rng.randn(M, 1, Da)
            act = old_mean + np.exp(old_ls) * rng.randn(M, N, Da)
            adv = rng.randn(M, N)
            f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
            obs, act, adv, old_mean, old_ls = f(obs), f(act), f(adv), f(old_mean), f(old_ls)
            nvm = nv if nv is not None else [N] * M
            self.cpus.append([dict(obs=obs[m:m + 1, :n], act=act[m:m + 1, :n], adv=adv[m:m + 1, :n], mean=old_mean[m:m + 1, :n],
                                   log_std=np.broadcast_to(old_ls[m:m + 1], (1, n, Da))) for m, n in enumerate(nvm)])
            if nv is not None:
                ph = RaggedPhaseData([[n] for n in nv], Do, Da, torch.device('cuda'))
                assert ph.N == N
                for m, n in enumerate(nv):
                    obs[m, n:] = 1e3; act[m, n:] = -50.0; adv[m, n:] = 1e4; old_mean[m, n:] = 7.0
            else:
                ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
            ph.obs.copy_(torch.from_numpy(obs)); ph.act.copy_(torch.from_numpy(act)); ph.mean.copy_(torch.from_numpy(old_mean))
            ph.log_std.copy_(torch.from_numpy(old_ls[:, 0]))
            ph.adv = torch.from_numpy(adv).cuda()
            self.phases.append(ph)
        if c.explore:
            self.coeff = rng.randn(M).astype(np.float32)
            self.phases[-1].adj_avg_rewards_mean = torch.from_numpy(self.coeff).cuda()
        if c.algo == 'promp':
            self._nudge_clip_ties()

    def data(self, m):
        out = []
        for s, per in enumerate(self.cpus):
            d = {k: torch.from_numpy(np.ascontiguousarray(v)).double() for k, v in per[m].items()}
            if self.c.explore and s == self.c.S1:
                d['adj_avg_rewards'] = torch.full_like(d['adv'], float(self.coeff[m]))
            out.append(d)
        return out

    def _nudge_clip_ties(self):
        """Outer samples whose float64 ratio lies within 1e-5 of 1 +- clip_eps get a zero advantage (float32 may take the other
        branch of the clipped objective)."""
        adv_dev = self.phases[-1].adv.cpu().numpy()
        a64 = torch.from_numpy(self.alpha).double()
        for m in range(self.c.M):
            d = self.data(m)
            cur = torch.from_numpy(self.theta).double().view(1, -1).requires_grad_(True)
            clip0 = self.pol.min_log_std
            for s in range(self.c.S1):
                cur = th.adapt_sym(cur, d[s], self.dims, a64, min_log_std=clip0)[0].detach().requires_grad_(True)
                clip0 = None
            with torch.no_grad():
                mean, ls = th.dist_info(cur, d[-1]['obs'], self.dims, clip0)
                r = th.likelihood_ratio(d[-1]['act'], d[-1]['mean'], d[-1]['log_std'], mean, ls).numpy()[0]
            tie = (np.abs(r - (1 - po.CLIP_EPS)) < 1e-5) | (np.abs(r - (1 + po.CLIP_EPS)) < 1e-5)
            self.cpus[-1][m]['adv'] = self.cpus[-1][m]['adv'].copy()
            self.cpus[-1][m]['adv'][0, tie] = 0.0
            adv_dev[m, :len(tie)][tie] = 0.0
        self.phases[-1].adv.copy_(torch.from_numpy(adv_dev))

    def oracle(self):
        """float64 d objective / d theta and d objective / d alpha, task means [P_logical] each."""
        c, algo = self.c, self.algo
        kind = 'promp' if c.algo == 'promp' else 'vpg'
        coeff = list(algo.inner_kl_coeff) if c.algo == 'promp' else None
        gt, ga = 0.0, 0.0
        for m in range(c.M):
            t64 = torch.tensor(self.theta, dtype=torch.float64, requires_grad=True)
            a64 = torch.tensor(self.alpha, dtype=torch.float64, requires_grad=True)
            obj, _, _ = th.meta_objective(t64, self.data(m), self.dims, a64, kind, po.CLIP_EPS, coeff,
                                          min_log_std=self.pol.min_log_std, exploration=c.explore)
            a, b = torch.autograd.grad(obj, (t64, a64))
            gt, ga = gt + a.numpy(), ga + b.numpy()
        return gt / c.M, ga / c.M

    def run(self):
        """[theta; alpha] gradient (task mean, float32, device layout) of one evaluation through the algorithm."""
        from promp_b200 import _lib
        from test_chain_plans import chain_options
        algo, P = self.algo, self.pol.num_params
        with chain_options(self.c.chain):
            res = algo._objective_pass(self.phases, want_grad=True)          # reduce=True: the [2P] gradient
            torch.cuda.synchronize()
        g = res['grad'].clone()
        assert g.shape == (2 * P,)
        if self.c.algo == 'promp':        # the fused path's reduce must agree bit for bit
            with chain_options(self.c.chain):
                res = algo._objective_pass(self.phases, want_grad=True, reduce=False)
                flat = torch.empty(2 * P, dtype=torch.float32, device='cuda')
                lam = _lib.ptr_array([a for a, _ in res['sgd_pairs']])
                gg = _lib.ptr_array([b for _, b in res['sgd_pairs']])
                _lib.call('promp_reduce_tasks_sgd', self.c.M, P, _lib.ptr(res['grad_tasks']), len(res['sgd_pairs']), lam, gg,
                          1.0 / self.c.M, _lib.ptr(flat), _lib.stream())
                torch.cuda.synchronize()
            assert torch.equal(flat, g), self.c.cid + ': promp_reduce_tasks_sgd differs from the reduce=True pass'
        return g


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c.cid for c in CASES])
def test_theta_and_alpha_gradients_against_float64(case):
    po._cuda()
    setup = Setup(case)
    g1 = setup.run()
    g2 = setup.run()
    assert torch.equal(g1, g2), case.cid + ': not run-to-run bit-identical'
    P, pol = setup.pol.num_params, setup.pol
    got = g1.cpu().numpy()
    mask = np.ones(P, dtype=bool)
    mask[pol._pad_index_np] = False
    assert np.all(got[:P][mask] == 0.0) and np.all(got[P:][mask] == 0.0), case.cid + ': pad entries are not 0.0'
    want_t, want_a = setup.oracle()
    H = case.hidden
    po.assert_blocks(case.cid + ' theta-gradient', pol.unpad_flat(got[:P])[None], want_t[None], case.Do, case.Da, H)
    po.assert_blocks(case.cid + ' alpha-gradient', pol.unpad_flat(got[P:])[None], want_a[None], case.Do, case.Da, H)


@pytest.mark.gpu
@pytest.mark.parametrize('chain', [-1, 0])
def test_alpha_equal_to_inner_lr_matches_the_scalar_path(chain):
    """alpha = inner_lr everywhere: _adapt is bit-identical to the scalar path (one launch per stage at this size), and the
    theta meta-gradient agrees with the scalar algorithm's within 1e-5."""
    from promp_b200.meta_algos import ProMP
    from test_chain_plans import chain_options
    po._cuda()
    setup = Setup(Case('s2', 'promp', 2, 2, 2, 64, M=4, N=300, chain=chain), alpha_scale=0.0)
    assert bool((setup.algo.alpha == np.float32(0.1)).all())
    fixed = ProMP(policy=setup.pol, inner_lr=0.1, meta_batch_size=4, num_inner_grad_steps=2, num_ppo_steps=1,
                  clip_eps=po.CLIP_EPS, init_inner_kl_penalty=5e-3, adaptive_inner_kl_penalty=False)
    out = []
    with chain_options(chain):
        for algo in (fixed, setup.algo):
            setup.pol.switch_to_pre_update()
            algo.adapt_phase(setup.phases[0])
            out.append((algo.last_inner_grad.clone(), setup.pol.theta_tasks.clone()))
            setup.pol.switch_to_pre_update()
        torch.cuda.synchronize()
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    P = setup.pol.num_params
    with chain_options(chain):
        fixed._adapt_cache = None
        gf = fixed._objective_pass(setup.phases, want_grad=True)['grad']
        gt = setup.algo._objective_pass(setup.phases, want_grad=True)['grad'][:P]
        torch.cuda.synchronize()
    assert float((gf - gt).norm() / gf.norm()) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize('algo_kind', ['promp', 'vpg'])
def test_one_adam_step_over_theta_and_alpha(algo_kind):
    """optimize_policy with one Adam epoch equals a float32 torch restatement of TF1 Adam over [theta; alpha] applied to the
    [2P] gradient of the same evaluation (ProMP: fused meta-update launch; VPG-MAML: reduce + Adam)."""
    po._cuda()
    setup = Setup(Case('adam', algo_kind, 2, 2, 2, 64))
    algo, pol, P = setup.algo, setup.pol, setup.pol.num_params
    g = setup.run()
    th0, a0 = pol.theta.clone(), algo.alpha.clone()
    adam = th.TF1Adam(2 * P, lr=1e-3)
    want = adam.step(torch.cat([th0, a0]).cpu(), g.cpu())
    for _ in range(2):       # the second step runs at the updated (theta, alpha) with persistent slots
        algo.optimizer.optimize(algo, setup.phases)
        if _ == 0:
            torch.cuda.synchronize()
            got = torch.cat([pol.theta, algo.alpha]).cpu()
            assert torch.equal(algo.optimizer.last_grad_full.cpu(), g.cpu())
            assert int(algo.optimizer.step.item()) == 1
            np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-6, atol=1e-9)
            assert not torch.equal(algo.alpha, a0)
    assert int(algo.optimizer.step.item()) == 2


def _trainer(M=4, E=3, H=30, n_itr=2, graph=False, seed=5):
    from promp_b200.envs import normalize, MetaPointEnvCorner
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    np.random.seed(seed)
    env = normalize(MetaPointEnvCorner(reward_type='dense'))        # sparse rewards leave short runs without an outer gradient
    policy = MetaGaussianMLPPolicy(name='p', obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-2, num_ppo_steps=3,
                 trainable_inner_step_size=True)
    tr = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=n_itr, num_inner_grad_steps=1,
                 use_cuda_graph=graph)
    return policy, algo, tr


@pytest.mark.gpu
def test_graph_mode_is_bit_identical_across_runs_and_trains_alpha():
    from promp_b200.utils import logger
    po._cuda()
    logger.set_quiet(True)
    out = []
    for _ in range(2):
        policy, algo, tr = _trainer(graph=True, n_itr=3)
        assert tr.graph_capturable()
        a0 = algo.alpha.clone()
        tr.train()
        out.append((policy.theta.clone(), algo.alpha.clone(), algo.optimizer.m_alpha.clone()))
        assert not torch.equal(algo.alpha, a0) and int(algo.optimizer.step.item()) == 9
    assert all(torch.equal(a, b) for a, b in zip(*out))


@pytest.mark.gpu
def test_captured_optimize_phases_equals_eager():
    """A captured ProMP optimize_phases replays to exactly what the eager call computes from the same state."""
    po._cuda()
    setup = Setup(Case('graph', 'promp', 1, 2, 2, 64))
    algo, pol = setup.algo, setup.pol
    algo.optimize_phases(setup.phases, want_terms=False)          # warm-up: allocations and one-time uploads
    torch.cuda.synchronize()
    state = [t.clone() for t in [pol.theta, algo.alpha] + algo.optimizer.slots()]
    live = [pol.theta, algo.alpha] + algo.optimizer.slots()
    algo.optimize_phases(setup.phases, want_terms=False)
    torch.cuda.synchronize()
    eager = [t.clone() for t in live]
    for d, s in zip(live, state):
        d.copy_(s)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, capture_error_mode='thread_local'):
            algo.optimize_phases(setup.phases, want_terms=False)
    torch.cuda.current_stream().wait_stream(side)
    for d, s in zip(live, state):
        d.copy_(s)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, live))


@pytest.mark.gpu
def test_snapshot_restore_and_continue_equals_the_uninterrupted_run(tmp_path):
    from promp_b200.utils import logger
    po._cuda()
    try:
        logger.configure(dir=str(tmp_path / 'a'), format_strs=['json'], snapshot_mode='all')
        policy, algo, tr = _trainer(n_itr=3)
        tr.train()
        full = (policy.theta.clone(), algo.alpha.clone())
        snap = logger.load_snapshot(os.path.join(str(tmp_path / 'a'), 'itr_1.pkl'))
        assert 'alpha' in snap['promp_b200_state'] and 'm_alpha' in snap['promp_b200_state']['optimizer']
        logger.configure(dir=str(tmp_path / 'b'), format_strs=['json'], snapshot_mode='none')
        policy2, algo2, tr2 = _trainer(n_itr=3, seed=11)
        # the sampler's numpy draws continue from where the uninterrupted run was after iteration 1
        policy3, algo3, tr3 = _trainer(n_itr=2)
        tr3.train()
        state = np.random.get_state()
        assert tr2.restore(snap) == 2
        np.random.set_state(state)
        tr2.sampler._phase_counter = tr3.sampler._phase_counter
        tr2.train()
        assert torch.equal(policy2.theta, full[0]) and torch.equal(algo2.alpha, full[1])
    finally:
        logger.reset()


@pytest.mark.gpu
@pytest.mark.parametrize('algo_kind', ['promp', 'vpg'])
def test_task_shards_sum_to_the_one_process_gradient(algo_kind, monkeypatch):
    """Tasks split as a task_shard=(r, 2) run splits them: each shard's algorithm sees its half of the tasks and scales by
    1 / (M_local * world).  Run one after another on one GPU, the shards' [theta; alpha] gradients sum to the one-process
    gradient (to float32 reassociation: the per-task sums run on a different launch geometry)."""
    from promp_b200.meta_algos import ProMP, VPGMAML
    from promp_b200.meta_algos import base as base_mod
    from promp_b200.samplers.device_data import PhaseData
    po._cuda()
    setup = Setup(Case('shard', algo_kind, 2, 2, 2, 64, M=4))
    full = setup.run()
    monkeypatch.setattr(base_mod, 'world_size', lambda: 2)
    total = torch.zeros_like(full)
    for r in range(2):
        lo, hi = 2 * r, 2 * r + 2
        kw = dict(policy=setup.pol, inner_lr=0.1, meta_batch_size=2, num_inner_grad_steps=2, trainable_inner_step_size=True)
        algo = ProMP(num_ppo_steps=1, clip_eps=po.CLIP_EPS, init_inner_kl_penalty=5e-3, adaptive_inner_kl_penalty=False, **kw) \
            if algo_kind == 'promp' else VPGMAML(**kw)
        algo.alpha.copy_(setup.algo.alpha)
        phases = []
        for ph in setup.phases:
            q = PhaseData(2, 1, ph.N, 2, 2, torch.device('cuda'))
            for k in ('obs', 'act', 'mean', 'log_std'):
                getattr(q, k).copy_(getattr(ph, k)[lo:hi])
            q.adv = ph.adv[lo:hi].contiguous()
            phases.append(q)
        total += algo._objective_pass(phases, want_grad=True)['grad']
    torch.cuda.synchronize()
    P = setup.pol.num_params
    for half in (slice(0, P), slice(P, 2 * P)):
        assert float((total[half] - full[half]).norm() / full[half].norm()) < 1e-6
