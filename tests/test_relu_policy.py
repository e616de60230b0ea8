"""Policies with ReLU hidden layers (MetaGaussianMLPPolicy(hidden_nonlinearity='relu' / tf.nn.relu / torch.relu)).

The oracle is the one of test_policy_oracle.py (float64 autograd over oracle/tf_half.py) with the policy forward
`tf_half.dist_info` replaced, for the tests of this module, by the same two-layer MLP with ReLU hidden layers.  torch's
ReLU backward, like TensorFlow's ReluGrad, passes no gradient at 0, which is what the kernels do.  That oracle is pinned
to the reference's UNMODIFIED graph code run with hidden_nonlinearity=tf.nn.relu (tests/golden/tf_half_relu.npz, written
by tools/make_relu_golden.py): inner adapt step, ProMP / TRPO-MAML / VPG-MAML objectives and meta-gradients, and the
finite-difference Hessian-vector product of TRPO-MAML.

CPU tests: the oracle against the golden outputs, the oracle HVP against central differences, the `hidden` flag of the
C ABI.  GPU tests (-m gpu): every policy kernel family with the ReLU activation against the float64 oracle at the 1e-4
per-(task, block) bar, the fused rollout, the dataflow chain, Trainer.train() and pickling.
"""
import math
import os
import pickle

import numpy as np
import pytest
import torch

import test_policy_oracle as po
from oracle import tf_half as th
from oracle import tf_cases

TANH_DIST_INFO = th.dist_info


def relu_dist_info(theta, obs, dims, min_log_std=None):
    """tf_half.dist_info with ReLU hidden layers (policies/networks/mlp.py with hidden_nonlinearity=tf.nn.relu)."""
    W0, b0, W1, b1, W2, b2, ls = th.split_params(theta, *dims)
    h = torch.relu(torch.matmul(obs, W0) + b0.unsqueeze(-2))
    h = torch.relu(torch.matmul(h, W1) + b1.unsqueeze(-2))
    mean = torch.matmul(h, W2) + b2.unsqueeze(-2)
    if min_log_std is not None:
        ls = torch.clamp(ls, min=min_log_std)
    return mean, ls


@pytest.fixture(autouse=True)
def relu_oracle(monkeypatch):
    """Every oracle function of oracle/tf_half.py (and the Case / oracle helpers of test_policy_oracle.py built on them)
    evaluates the ReLU policy inside the tests of this module."""
    monkeypatch.setattr(th, 'dist_info', relu_dist_info)


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


# ================================================================================================ CPU: oracle vs reference graph
_GOLD = None


def _gold(golden_dir):
    global _GOLD
    if _GOLD is None:
        _GOLD = np.load(os.path.join(golden_dir, 'tf_half_relu.npz'))
    return _GOLD


GOLDEN_CASES = ('promp_small', 'promp_cheetah', 'promp_s3', 'trpo_small', 'vpg_small')


def _oracle_data(case, dt):
    N = case['N']
    return [dict(obs=torch.tensor(p['obs'], dtype=dt), act=torch.tensor(p['act'], dtype=dt),
                 adv=torch.tensor(p['adv'], dtype=dt), mean=torch.tensor(p['mean'], dtype=dt),
                 log_std=torch.tensor(p['log_std'], dtype=dt)[:, None, :].expand(-1, N, -1),
                 adj_avg_rewards=torch.tensor(p['adj_avg_rewards'], dtype=dt)) for p in case['phases']]


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_relu_oracle_matches_reference_graph(golden_dir, name):
    """The float64 ReLU oracle == the unmodified reference graph with hidden_nonlinearity=tf.nn.relu, evaluated in float64:
    adapted parameters, objective, KLs, second-order meta-gradient, and for TRPO-MAML the KL gradient and the
    Hessian-vector product of the KL.  (The fixture stores vectors as float32: 6e-8 relative, far below the 1e-6 bar.)"""
    G = _gold(golden_dir)
    case = tf_cases.make_case(name)
    dt, tol = torch.float64, 1e-6
    # the reference's inner_lr is a float32 constant: with ReLU, the float64 value 0.1 can move an adapted pre-activation
    # that lies within 1e-8 of 0 across it, so the oracle takes the same float32-rounded step
    lr = float(np.float32(0.1))
    pre = name + '/f64/'
    keep = G[name + '/keep_tasks']
    dims = (case['Do'], case['Da'], (case['hidden'],) * 2)
    data = _oracle_data(case, dt)
    inner = case.get('inner_type', 'likelihood_ratio')
    theta = torch.tensor(case['theta'], dtype=dt)
    cur = theta[None].expand(case['M'], -1).contiguous()
    for s in range(case['S'] - 1):
        cur = th.adapt(cur, data[s], dims, lr, inner)
        delta = cur.numpy() - case['theta'].astype(np.float64)
        assert rel_err(delta[keep], G[pre + 'adapt%d_delta' % s]) < tol
        np.testing.assert_allclose(np.sqrt((delta ** 2).sum(1)), G[pre + 'adapt%d_delta_norm' % s], rtol=tol)
    t = theta.clone().requires_grad_(True)
    obj, ikl, okl = th.meta_objective(t, data, dims, lr, case['algo'], 0.3, [5e-4] * (case['S'] - 1), inner)
    (g,) = torch.autograd.grad(obj, t)
    assert abs(float(obj.detach()) - float(G[pre + 'loss'])) <= 1e-9 + tol * abs(float(G[pre + 'loss']))
    assert rel_err(g.numpy(), G[pre + 'grad']) < tol
    if case['algo'] == 'promp':
        np.testing.assert_allclose(ikl.detach().numpy(), G[pre + 'inner_kl'], rtol=10 * tol, atol=1e-12)
    if case['algo'] in ('promp', 'trpo'):
        assert abs(float(okl.detach()) - float(G[pre + 'outer_kl'])) <= 1e-12 + 10 * tol * abs(float(G[pre + 'outer_kl']))
    if case['algo'] == 'trpo':
        def kl_grad(th_np):
            t = torch.as_tensor(th_np, dtype=dt).clone().requires_grad_(True)
            (gk,) = torch.autograd.grad(th.meta_objective(t, data, dims, lr, 'trpo', inner_type=inner)[2], t)
            return gk.numpy()
        assert rel_err(kl_grad(case['theta']), G[pre + 'kl_grad']) < tol
        gw = G[pre + 'grad'].astype(np.float64)
        x, eps, th64 = gw / np.linalg.norm(gw), float(np.float32(1e-5)), case['theta'].astype(np.float64)
        hx = (kl_grad(th64 + eps * x) - kl_grad(th64 - eps * x)) / (2 * eps)
        assert rel_err(hx, G[pre + 'hx']) < 1e-4


def _active(theta, obs, dims):
    """The ReLU units that are on (pre-activation > 0) in both hidden layers."""
    W0, b0, W1, b1 = th.split_params(theta, *dims)[:4]
    z1 = torch.matmul(obs, W0) + b0.unsqueeze(-2)
    z2 = torch.matmul(torch.relu(z1), W1) + b1.unsqueeze(-2)
    return torch.cat([z1 > 0, z2 > 0], -1)


def test_relu_hvp_oracle_matches_central_differences():
    """The exact HVP (double backward through the ReLU oracle) == central differences of its gradient, at inputs where no
    pre-activation changes sign inside the difference step (ReLU is linear between its kinks)."""
    case = po.Case(5, 3, 32, 3, 200, seed=21)
    vec = case.vec()
    eps = 1e-6
    t0, v, obs = case.theta_t(), torch.from_numpy(vec).double(), case.data()['obs']
    on = _active(t0, obs, case.dims)
    assert 0.2 < float(on.double().mean()) < 0.8
    assert torch.equal(on, _active(t0 + eps * v, obs, case.dims)) and torch.equal(on, _active(t0 - eps * v, obs, case.dims))
    for kind in ('ratio', 'loglik'):
        want = case.hvp_delta(kind, vec, 1.0, 0.0).numpy()
        fd = po._central_difference_hvp(case, kind, vec, eps=eps).numpy()
        po.assert_blocks('central differences ' + kind, fd, want, 5, 3, 32)


def test_relu_and_tanh_oracles_differ(monkeypatch):
    """The same weights under tanh and ReLU give different gradients and HVPs far outside the bar: a kernel that ran the
    wrong activation fails the GPU tests."""
    case = po.Case(2, 2, 32, 2, 100, seed=3)
    vec = case.vec()
    relu = case.grad('ratio')[0].numpy(), case.hvp_delta('ratio', vec, 0.1, 0.0).numpy()
    monkeypatch.setattr(th, 'dist_info', TANH_DIST_INFO)
    tanh = case.grad('ratio')[0].numpy(), case.hvp_delta('ratio', vec, 0.1, 0.0).numpy()
    assert not po.blocks_pass(relu[0], tanh[0], 2, 2, 32) and not po.blocks_pass(relu[1], tanh[1], 2, 2, 32)


def test_activation_names():
    """hidden_nonlinearity accepted by MetaGaussianMLPPolicy: a name, or a callable recognised by its __name__ (the
    tf_shim placeholders that run scripts pass, torch.relu, F.relu)."""
    import importlib.util
    import torch.nn.functional as F
    from promp_b200.policies.meta_gaussian_mlp_policy import _activation_name
    shim = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'promp_b200', 'tf_shim', 'tensorflow',
                        '__init__.py')
    spec = importlib.util.spec_from_file_location('promp_tf_shim', shim)      # not as `tensorflow`: oracle/stubs_tf owns that name
    tf = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tf)
    for fn in ('relu', torch.relu, F.relu, tf.nn.relu):
        assert _activation_name(fn) == 'relu', fn
    for fn in (None, 'tanh', torch.tanh, tf.tanh):
        assert _activation_name(fn) == 'tanh', fn
    for fn in ('sigmoid', torch.sigmoid, F.elu, 'Relu', 3):
        assert _activation_name(fn) is None, fn


def test_abi_hidden_flag():
    """PROMP_ACT_RELU in the `hidden` argument: num_params / layout / workspace sizes unchanged, unknown bits and ReLU at an
    unsupported width rejected (before any device work: these calls are safe without a GPU)."""
    from promp_b200 import _lib
    lib = _lib.load()
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'promp_b200.h')).read()
    assert '#define PROMP_ACT_RELU 0x%x' % _lib.ACT_RELU in header
    assert '#define PROMP_HIDDEN_WIDTH_MASK 0x%X' % _lib.HIDDEN_WIDTH_MASK in header
    R = _lib.ACT_RELU
    for Do, Da in ((2, 2), (17, 6), (5, 3), (19, 8)):
        for h in (32, 64):
            assert lib.promp_num_params(Do, Da, h | R) == lib.promp_num_params(Do, Da, h) == th.num_params(Do, Da, (h, h))
            assert _lib.policy_layout(Do, Da, h | R) == _lib.policy_layout(Do, Da, h)
            assert lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h | R) == lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h)
            assert (lib.promp_policy_workspace_bytes_padded(40, 2000, Do, Da, h | R)
                    == lib.promp_policy_workspace_bytes_padded(40, 2000, Do, Da, h))
    assert lib.promp_num_params(2, 2, 300) == th.num_params(2, 2, (300, 300))    # other values keep their meaning
    with pytest.raises(_lib.PrompLibraryError, match='unknown flag bits'):
        _lib.policy_layout(2, 2, 64 | 0x200)
    with pytest.raises(_lib.PrompLibraryError, match='ReLU policies are built for hidden 32 or 64'):
        _lib.policy_layout(2, 2, 48 | R)
    # entry points: a non-null dummy address for every pointer; the hidden check fails before anything is launched
    dummy = 16
    for hidden, msg in ((64 | 0x400, 'unknown flag bits'), (16 | R, 'ReLU policies are built for hidden 32 or 64'),
                        (-64, 'unknown flag bits')):
        assert lib.promp_policy_forward(2, 2, hidden, 1, 1, dummy, 0, dummy, dummy, None) == -1
        assert msg in _lib.last_error()
        assert lib.promp_policy_forward_padded(5, 3, hidden, 1, 1, dummy, 0, dummy, dummy, None) == -1
        assert msg in _lib.last_error()
        assert lib.promp_rollout(_lib.ENV_POINT_CORNER, 0, 0.5, 1, 1, 1, 4, hidden, dummy, 0, dummy, None, None, 1, 1, None, 1,
                                 -13.8, dummy, dummy, dummy, dummy, dummy, None, dummy, None, None) == -1
        assert msg in _lib.last_error()
        assert lib.promp_rollout_early_term(_lib.ENV_POINT, 1, 1, 1, 8, 4, hidden, dummy, 0, dummy, None, None, 1, 1, None, 1,
                                            -13.8, dummy, dummy, dummy, dummy, dummy, dummy, None) == -1
        assert msg in _lib.last_error()
    import ctypes
    stage = _lib.PolicyStage(kind=0, N=100)          # read on the host only
    for fn in (lib.promp_policy_chain_workspace_bytes, lib.promp_policy_chain_num_launches):
        assert fn(2, 2, 64 | R, 4, 1, ctypes.byref(stage)) == fn(2, 2, 64, 4, 1, ctypes.byref(stage)) > 0
        assert fn(2, 2, 64 | 0x800, 4, 1, ctypes.byref(stage)) == -1


# ================================================================================================================ GPU
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from promp_b200 import _lib
    _lib.require_cuda()


def _relu_policy(Do, Da, hidden_sizes, M, nonlinearity='relu'):
    from promp_b200.policies import MetaGaussianMLPPolicy
    return MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=hidden_sizes,
                                 hidden_nonlinearity=nonlinearity)


class ReluLauncher(po.Launcher):
    """test_policy_oracle.Launcher on a ReLU policy: every call passes `policy.hidden_arg` (width | PROMP_ACT_RELU)."""

    def __init__(self, case):
        orig = po._policy
        po._policy = lambda c: _relu_policy(c.Do, c.Da, (c.hidden, c.hidden), c.M)
        try:
            super(ReluLauncher, self).__init__(case)
        finally:
            po._policy = orig
        assert self.pol.hidden_arg == self.pol.hidden | self.lib.ACT_RELU

    def grad(self, kind, obj_scale=1.0, kl_coeff=0.0, clip=1, sgd_lr=0.1):
        c, M = self.case, self.case.M
        grad = torch.full((M, self.P), float('nan'), device='cuda')
        newp = torch.full((M, self.P), float('nan'), device='cuda')
        stats = torch.full((M, 4), float('nan'), device='cuda')
        p = self.lib.ptr
        self.lib.call(self.pol.entries['grad_ex'], c.Do, c.Da, self.pol.hidden_arg, M, c.N, p(self.n_valid), p(self.params),
                      self.stride, p(self.obs), p(self.act), p(self.adv), p(self.mean), p(self.old_ls), int(c.ls_per_sample),
                      po.OBJ[kind], float(obj_scale), po.CLIP_EPS, float(kl_coeff), int(clip), float(c.min_log_std), p(grad),
                      p(newp), float(sgd_lr), p(stats), None, None, None, None, p(self.ws), self.ws.numel() * 4, self.lib.stream())
        torch.cuda.synchronize()
        return grad, newp, stats

    def hvp(self, kind, vec, inner_lr=0.1, kl_coeff=5e-4, clip=1):
        c, M = self.case, self.case.M
        v = torch.from_numpy(self.pol.pad_flat(vec)).cuda()
        out = torch.full((M, self.P), float('nan'), device='cuda')
        stats = torch.full((M, 4), float('nan'), device='cuda')
        p = self.lib.ptr
        self.lib.call(self.pol.entries['hvp_ragged'], c.Do, c.Da, self.pol.hidden_arg, M, c.N, p(self.n_valid), p(self.params),
                      self.stride, p(self.obs), p(self.act), p(self.adv), p(self.mean), p(self.old_ls), int(c.ls_per_sample),
                      po.OBJ[kind], float(inner_lr), float(kl_coeff), int(clip), float(c.min_log_std), p(v), p(out), p(stats),
                      p(self.ws), self.ws.numel() * 4, self.lib.stream())
        torch.cuda.synchronize()
        return v, out, stats

    def forward(self):
        c, M = self.case, self.case.M
        mean = torch.full((M, c.N, c.Da), float('nan'), device='cuda')
        p = self.lib.ptr
        self.lib.call(self.pol.entries['forward'], c.Do, c.Da, self.pol.hidden_arg, M, c.N, p(self.params), self.stride,
                      p(self.obs), p(mean), self.lib.stream())
        torch.cuda.synchronize()
        return mean.cpu().numpy()


def _relu_kernels(path, Do, Da, hidden):
    return [k.replace('_kernel<', '_relu_kernel<') for k in po._expected_kernels(path, Do, Da, hidden)]


SHAPES = po.EXACT_SHAPES + po.BUCKET_SHAPES


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da', SHAPES, ids=['%dx%d' % s for s in SHAPES])
@pytest.mark.parametrize('path', po.PATHS)
def test_relu_kernels_match_oracle(path, Do, Da):
    """Gradient (RATIO + KL, CLIP, LOGLIK), HVP and forward of every kernel path at every exact and bucket shape against the
    float64 ReLU oracle; N = 300 fills no 64- or 128-sample tile exactly; the kernels the profiler records are the path's
    ReLU kernels."""
    _cuda()
    hidden = 32 if path == 'h32' else 64
    case = po.Case(Do, Da, hidden, 3, 300, seed=200 + Do * 10 + Da)
    with po._path(path):
        L = ReluLauncher(case)
        what = 'relu %s %dx%d' % (path, Do, Da)
        po.check_grad(L, what, 'ratio', kl_coeff=0.1)
        po.check_grad(L, what, 'clip', kl_coeff=0.2)
        po.check_hvp(L, what, 'ratio')
        po.check_hvp(L, what, 'loglik')
        mu, _ = relu_dist_info(case.theta_t(), case.data()['obs'], case.dims)
        np.testing.assert_allclose(L.forward(), mu.numpy(), rtol=1e-4, atol=1e-5 * float(np.abs(mu.numpy()).max()))
        names = po._kernels_run_by(lambda: (L.grad('ratio'), L.hvp('ratio', case.vec())))
    # Every policy kernel the profiler recorded is one this path must run, with the ReLU activation.  (A session does not
    # always record every launch of a long test run, so a kernel missing from the record is not a failure.)
    expected = _relu_kernels(path, Do, Da, hidden)
    for k in set(k for k in (names or []) if 'policy_' in k):
        assert any(name in k for name in expected), (k, expected)


@pytest.mark.gpu
@pytest.mark.parametrize('path', ['cuda', 'tc512', 'h32'])
def test_relu_ragged_shared_and_deterministic(path):
    """Ragged n_valid with poisoned padding, per-task and shared parameters, a binding log_std clip; two launches give the
    same bits."""
    _cuda()
    hidden = 32 if path == 'h32' else 64
    M = 4
    cases = [po.Case(2, 2, hidden, M, 257, seed=7, n_valid=[257, 1, 130, 64]),
             po.Case(17, 6, hidden, M, 200, seed=8, shared=True, ls=po._binding_ls(1, 6, -0.3, 9), min_log_std=-0.3),
             po.Case(5, 3, hidden, M, 129, seed=9, ls_per_sample=True)]
    with po._path(path):
        for case in cases:
            L = ReluLauncher(case)
            what = 'relu %s %dx%d' % (path, case.Do, case.Da)
            po.check_grad(L, what, 'ratio', kl_coeff=0.1)
            po.check_hvp(L, what, 'ratio')
            g1, _, s1 = L.grad('clip', kl_coeff=0.1)
            g2, _, s2 = L.grad('clip', kl_coeff=0.1)
            vec = case.vec()
            _, o1, _ = L.hvp('ratio', vec)
            _, o2, _ = L.hvp('ratio', vec)
            assert torch.equal(g1, g2) and torch.equal(s1[:, :3], s2[:, :3]) and torch.equal(o1, o2), what


@pytest.mark.gpu
def test_relu_tensor_cores_match_cuda_cores():
    """Hidden 64: the tensor-core gradient / HVP (3xTF32) against the CUDA-core kernels on the same inputs."""
    _cuda()
    for Do, Da in ((2, 2), (17, 6), (19, 8)):
        case = po.Case(Do, Da, 64, 3, 333, seed=50 + Do)
        vec = case.vec()
        res = {}
        for path in ('cuda', 'tc256', 'tc512'):
            with po._path(path):
                L = ReluLauncher(case)
                res[path] = (L.logical(L.grad('ratio', kl_coeff=0.1)[0]),
                             L.pol.unpad_flat(L.hvp('ratio', vec)[1].cpu().numpy()).astype(np.float64) - vec)
        for path in ('tc256', 'tc512'):
            for k in range(2):
                po.assert_blocks('relu %s vs cuda %dx%d' % (path, Do, Da), res[path][k], res['cuda'][k], Do, Da, 64)


@pytest.mark.gpu
def test_relu_zero_padded_hidden_units():
    """hidden_sizes (16, 16) run on the hidden-32 kernels: the padded units output relu(0) = 0 and get exactly zero
    gradient and HVP."""
    _cuda()
    case = po.Case(2, 2, 16, 3, 150, seed=12)
    with po._path('cuda'):
        L = ReluLauncher(case)
        assert L.pol.hidden == 32 and L.pol.num_params > L.pol.num_params_logical
        po.check_grad(L, 'relu 16x16', 'ratio', kl_coeff=0.1)
        po.check_hvp(L, 'relu 16x16', 'ratio')


def _product_algo(case):
    from promp_b200.meta_algos import ProMP, TRPOMAML, VPGMAML
    H = tf_cases.HYPER
    M, S1 = case['M'], case['S'] - 1
    np.random.seed(1)
    policy = _relu_policy(case['Do'], case['Da'], (case['hidden'],) * 2, M)
    policy.set_params(tf_cases.unflatten(case['theta'], case['Do'], case['Da'], case['hidden']))
    if case['algo'] == 'promp':
        algo = ProMP(policy=policy, inner_lr=H['inner_lr'], meta_batch_size=M, num_inner_grad_steps=S1,
                     learning_rate=H['learning_rate'], num_ppo_steps=H['num_ppo_steps'], clip_eps=H['clip_eps'],
                     target_inner_step=0.01, init_inner_kl_penalty=H['init_inner_kl_penalty'], adaptive_inner_kl_penalty=False)
    elif case['algo'] == 'trpo':
        algo = TRPOMAML(policy=policy, step_size=H['step_size'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                        meta_batch_size=M, num_inner_grad_steps=S1)
    else:
        algo = VPGMAML(policy=policy, learning_rate=H['learning_rate'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                       meta_batch_size=M, num_inner_grad_steps=S1)
    return policy, algo


@pytest.mark.gpu
@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_relu_adapt_and_meta_gradient_match_reference_graph(golden_dir, name):
    """MAMLAlgo._adapt (SGD) and the second-order meta-gradient (S1 = 1 and 2) of a ReLU policy on the device against the
    unmodified reference graph with tf.nn.relu (float64 evaluation), at the 1e-4 bar.  ProMP / VPG-MAML: the dataflow
    chain and one launch per stage give the same gradient."""
    _cuda()
    from promp_b200 import _lib
    G = _gold(golden_dir)
    case = tf_cases.make_case(name)
    samples = tf_cases.reference_samples(case)
    pre = name + '/f64/'
    th0 = case['theta'].astype(np.float64)
    grads = {}
    # promp_policy_chain: the dataflow kernel (1) and one launch per stage (0), each on a fresh policy / algorithm
    for chain in ((1, 0) if case['algo'] != 'trpo' else (-1,)):
        _lib.set_option('chain', chain)
        try:
            policy, algo = _product_algo(case)
            policy.switch_to_pre_update()
            for s in range(case['S'] - 1):
                algo._adapt(samples[s])
                delta = policy.theta_tasks.cpu().numpy().astype(np.float64) - th0[None]
                want = G[pre + 'adapt%d_delta' % s]
                assert rel_err(delta[G[name + '/keep_tasks']], want) < 1e-4, rel_err(delta[G[name + '/keep_tasks']], want)
                np.testing.assert_allclose(np.sqrt((delta ** 2).sum(1)), G[pre + 'adapt%d_delta_norm' % s], rtol=1e-4)
            phases = [algo._phase_of(s) for s in samples]
            if case['algo'] == 'trpo':
                g_got = algo.eval_gradient(policy.theta, phases, 'loss')
                gk = algo.eval_gradient(policy.theta, phases, 'kl')
                assert rel_err(gk, G[pre + 'kl_grad']) < 1e-4, rel_err(gk, G[pre + 'kl_grad'])
                loss, _ = algo.eval_scalars(policy.theta, phases)
            else:
                res = algo._objective_pass(phases, want_grad=True)
                g_got = res['grad'].cpu().numpy().astype(np.float64)
                loss = algo.loss_terms(res).cpu().numpy()[0]
        finally:
            _lib.set_option('chain', -1)
        assert abs(float(loss) - float(G[pre + 'loss'])) <= 2e-6 + 1e-4 * abs(float(G[pre + 'loss'])), (chain, loss)
        assert rel_err(g_got, G[pre + 'grad']) < 1e-4, (chain, rel_err(g_got, G[pre + 'grad']))
        grads[chain] = g_got
    if len(grads) == 2:
        assert rel_err(grads[1], grads[0]) < 2e-5, rel_err(grads[1], grads[0])


# ------------------------------------------------------------------------------------------------ fused rollout
# (env kind, obs, act, task floats, early-terminating)
ROLLOUT_ENVS = dict(point_corner=(0, 2, 2, 2, False), point=(1, 2, 2, 1, True), cheetah=(2, 17, 6, 1, False),
                    swimmer=(6, 8, 2, 1, False), walker=(5, 17, 6, 2, True))


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', [64, 32])
@pytest.mark.parametrize('env', list(ROLLOUT_ENVS))
def test_relu_fused_rollout_teacher_forced(env, hidden):
    """promp_rollout / promp_rollout_early_term with a ReLU policy and fed noise: the recorded means against the float64
    ReLU policy evaluated on the kernel's own observations, and act = mean + eps * exp(log_std)."""
    _cuda()
    from promp_b200 import _lib
    kind, Do, Da, TD, early = ROLLOUT_ENVS[env]
    M, E, H = 3, 6, 40
    rng = np.random.RandomState(kind * 10 + hidden)
    dims = (Do, Da, (hidden, hidden))
    PL = th.num_params(*dims)
    theta = th.init_params(*dims, rng=rng).astype(np.float64)[None] + 0.1 * rng.randn(M, PL)
    theta[:, PL - Da:] = -0.5
    theta = theta.astype(np.float32)
    if kind == 2:
        task = rng.choice([-1.0, 1.0], size=(M, 1))
    elif kind == 5:
        task = np.stack([rng.uniform(0, 2, M), rng.randint(0, 2, M)], 1)
    else:
        task = rng.uniform(-1, 1, size=(M, TD))
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    T = 2 * H - 1 if early else H
    noise = rng.randn(M, E, T, Da).astype(np.float32)
    obs, act, mean = (torch.empty(M, E, T, n, device='cuda') for n in (Do, Da, Da))
    rew = torch.empty(M, E, T, device='cuda')
    done = torch.empty(M, E, T, dtype=torch.uint8, device='cuda')
    ls_out = torch.empty(M, Da, device='cuda')
    info = torch.zeros(3, M, E, T, device='cuda')
    p = _lib.ptr
    hidden_arg = hidden | _lib.ACT_RELU
    params, task_d, noise_d = dev(theta), dev(task), dev(noise)
    if early:
        _lib.call('promp_rollout_early_term', kind, 1, M, E, T, H, hidden_arg, p(params), PL, p(task_d), None, p(noise_d),
                  5, 1, None, 0, -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(ls_out), _lib.stream())
    else:
        _lib.call('promp_rollout', kind, 0 if kind != 0 else 1, 0.5, 1, M, E, H, hidden_arg, p(params), PL, p(task_d), None,
                  p(noise_d), 5, 1, None, 0, -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(info), p(ls_out), None,
                  _lib.stream())
    torch.cuda.synchronize()
    o, a, mu = obs.cpu().numpy(), act.cpu().numpy(), mean.cpu().numpy()
    if early:
        assert done.cpu().numpy().sum() >= M * E        # every slot finished at least one path and kept stepping after its reset
    want, _ = relu_dist_info(torch.from_numpy(theta).double(), torch.from_numpy(o.reshape(M, E * T, Do)).double(), dims)
    want = want.numpy().reshape(M, E, T, Da)
    np.testing.assert_allclose(mu, want, rtol=1e-4, atol=2e-5)
    sig = np.exp(theta[:, -Da:].astype(np.float64))[:, None, None, :]
    np.testing.assert_allclose(a, mu + noise * sig, rtol=1e-5, atol=1e-5)
    # the tanh kernel on the same inputs records different means: the flag selected the ReLU kernel
    _lib.call('promp_rollout_early_term' if early else 'promp_rollout',
              *((kind, 1, M, E, T, H, hidden, p(params), PL, p(task_d), None, p(noise_d), 5, 1, None, 0, -13.8, p(obs), p(act),
                 p(mean), p(rew), p(done), p(ls_out), _lib.stream()) if early else
                (kind, 0 if kind != 0 else 1, 0.5, 1, M, E, H, hidden, p(params), PL, p(task_d), None, p(noise_d), 5, 1, None, 0,
                 -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(info), p(ls_out), None, _lib.stream())))
    torch.cuda.synchronize()
    assert not np.allclose(mean.cpu().numpy()[:, :, 0], mu[:, :, 0])


# ------------------------------------------------------------------------------------------------ Trainer
def _train(kind, tmp_path, seed, graph=False):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnvCorner, HalfCheetahRandDirecEnv, Walker2DRandVelEnv
    from promp_b200.meta_algos import ProMP, TRPOMAML
    from promp_b200.meta_trainer import Trainer
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.utils import logger
    M, E, H = 4, 3, 30
    np.random.seed(seed)
    torch.manual_seed(seed)
    sampler_kw = {}
    if kind in ('point', 'trpo'):
        env = normalize(MetaPointEnvCorner(reward_type='dense'))    # sparse rewards give all-zero advantages at this size
    elif kind == 'cheetah':
        env = normalize(HalfCheetahRandDirecEnv())
    else:
        env = normalize(Walker2DRandVelEnv())
        sampler_kw = dict(reset_mode='device')
    Do, Da = int(np.prod(env.observation_space.shape)), int(np.prod(env.action_space.shape))
    policy = _relu_policy(Do, Da, (64, 64), M, nonlinearity=torch.relu)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H, **sampler_kw)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    if kind == 'trpo':
        algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, step_size=0.01)
    else:
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=3, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                      num_inner_grad_steps=1, use_cuda_graph=graph)
    if graph:
        assert trainer.graph_capturable()
    theta0 = policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='last')
        trainer.train()
        kv = logger.last_dump()
    finally:
        logger.reset()
    assert not torch.equal(policy.theta, theta0) and torch.isfinite(policy.theta).all()
    return policy, kv


@pytest.mark.gpu
@pytest.mark.parametrize('kind,graph', [('point', True), ('cheetah', True), ('trpo', False), ('walker', False)])
def test_relu_trainer_runs(kind, graph, tmp_path):
    """Three meta-iterations of Trainer.train() with a ReLU policy: ProMP in CUDA-graph mode (point, cheetah), TRPO-MAML,
    and the walker with device resets (early termination).  Every logged scalar is finite and the same seed gives the
    same results; the snapshot keeps the activation."""
    _cuda()
    policy, kv = _train(kind, tmp_path / 'a', seed=11, graph=graph)
    policy2, kv2 = _train(kind, tmp_path / 'b', seed=11, graph=graph)
    assert kv['Itr'] == 2
    for key in ('Step_0-AverageReturn', 'Step_1-AverageReturn', 'LossBefore', 'LossAfter'):
        assert key in kv, key
    assert all(np.isfinite(v) for k, v in kv.items() if isinstance(v, (float, int, np.floating)) and 'Time' not in k)
    assert torch.equal(policy.theta, policy2.theta)
    for k, v in kv.items():
        if 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert v == kv2[k], k
    from promp_b200.utils import logger
    snap = logger.load_snapshot(os.path.join(str(tmp_path / 'a'), 'params.pkl'))
    pol = snap['policy']
    assert pol.hidden_nonlinearity == 'relu' and pol.hidden_arg == policy.hidden_arg
    assert torch.equal(pol.theta, policy.theta)


@pytest.mark.gpu
def test_relu_policy_pickle_round_trip_and_rejections():
    _cuda()
    from promp_b200.policies import MetaGaussianMLPPolicy
    pol = _relu_policy(17, 6, (64, 64), 3, nonlinearity=torch.nn.functional.relu)
    assert pol.hidden_nonlinearity == 'relu' and pol.hidden_arg == 64 | 0x100
    pol2 = pickle.loads(pickle.dumps(pol))
    assert pol2.hidden_nonlinearity == 'relu' and pol2.hidden_arg == pol.hidden_arg and torch.equal(pol2.theta, pol.theta)
    # a state saved before the activation was stored loads as tanh
    state = pol.__getstate__()
    del state['init_args']['hidden_nonlinearity']
    old = MetaGaussianMLPPolicy.__new__(MetaGaussianMLPPolicy)
    old.__setstate__(state)
    assert old.hidden_nonlinearity == 'tanh' and old.hidden_arg == 64
    tanh_pol = _relu_policy(2, 2, (32, 32), 2, nonlinearity='tanh')
    assert tanh_pol.hidden_arg == tanh_pol.hidden == 32
    for bad in ('sigmoid', torch.sigmoid):
        with pytest.raises(NotImplementedError, match='tanh or relu'):
            _relu_policy(2, 2, (32, 32), 2, nonlinearity=bad)
    # get_actions (promp_policy_forward) with ReLU
    obs = [np.random.RandomState(m).randn(5, 17).astype(np.float32) for m in range(3)]
    _, infos = pol.get_actions(obs)
    theta = torch.from_numpy(pol.unpad_flat(pol.theta.cpu().numpy())).double()[None].expand(3, -1)
    want, _ = relu_dist_info(theta, torch.from_numpy(np.stack(obs)).double(), (17, 6, (64, 64)))
    got = np.stack([[infos[m][e]['mean'] for e in range(5)] for m in range(3)])
    np.testing.assert_allclose(got, want.numpy(), rtol=1e-4, atol=1e-5)
