"""Policies with a tanh output layer (MetaGaussianMLPPolicy(output_nonlinearity='tanh' / tf.tanh / torch.tanh)).

The oracle is the one of test_policy_oracle.py (float64 autograd over oracle/tf_half.py) with the policy forward
`tf_half.dist_info` replaced, for the tests of this module, by the two-layer MLP with mean = tanh(h2 W2 + b2), with tanh or
ReLU hidden layers.  That oracle is pinned to the reference's UNMODIFIED graph code run with output_nonlinearity=tf.tanh
(tests/golden/tf_half_otanh.npz, written by tools/make_otanh_golden.py): inner adapt step, ProMP / TRPO-MAML / VPG-MAML
objectives and meta-gradients, and the finite-difference Hessian-vector product of TRPO-MAML.

CPU tests: the oracle against the golden outputs, the oracle HVP against central differences, the `hidden` flag of the C
ABI, the constructor's names.  GPU tests (-m gpu): every policy kernel family with the tanh output against the float64
oracle at the 1e-4 per-(task, block) bar, the dataflow chain, the fused rollout, get_actions, Trainer.train() and pickling.
"""
import os
import pickle

import numpy as np
import pytest
import torch

import test_policy_oracle as po
from oracle import tf_half as th
from oracle import tf_cases

IDENTITY_DIST_INFO = th.dist_info


def otanh_dist_info_for(act):
    """tf_half.dist_info with `act` ('tanh' | 'relu') hidden layers and a tanh output layer (policies/networks/mlp.py with
    output_nonlinearity=tf.tanh)."""
    f = torch.relu if act == 'relu' else torch.tanh

    def dist_info(theta, obs, dims, min_log_std=None):
        W0, b0, W1, b1, W2, b2, ls = th.split_params(theta, *dims)
        h = f(torch.matmul(obs, W0) + b0.unsqueeze(-2))
        h = f(torch.matmul(h, W1) + b1.unsqueeze(-2))
        mean = torch.tanh(torch.matmul(h, W2) + b2.unsqueeze(-2))
        if min_log_std is not None:
            ls = torch.clamp(ls, min=min_log_std)
        return mean, ls
    return dist_info


DIST = dict(tanh=otanh_dist_info_for('tanh'), relu=otanh_dist_info_for('relu'))


@pytest.fixture(autouse=True)
def otanh_oracle(monkeypatch):
    """Every oracle function of oracle/tf_half.py evaluates the tanh-output policy (tanh hidden layers unless a test switches
    to ReLU with _use) inside the tests of this module."""
    monkeypatch.setattr(th, 'dist_info', DIST['tanh'])
    return monkeypatch


def _use(monkeypatch, act):
    monkeypatch.setattr(th, 'dist_info', DIST[act])


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


# ================================================================================================ CPU: oracle vs reference graph
_GOLD = None


def _gold(golden_dir):
    global _GOLD
    if _GOLD is None:
        _GOLD = np.load(os.path.join(golden_dir, 'tf_half_otanh.npz'))
    return _GOLD


# (hidden activation, case): the cases of tools/make_otanh_golden.py
GOLDEN_CASES = (('tanh', 'promp_small'), ('tanh', 'promp_cheetah'), ('tanh', 'promp_s3'), ('tanh', 'promp_h32'),
                ('tanh', 'trpo_small'), ('tanh', 'vpg_small'), ('relu', 'promp_small'), ('relu', 'vpg_small'))
GOLDEN_IDS = ['%s-%s' % c for c in GOLDEN_CASES]


def _oracle_data(case, dt):
    N = case['N']
    return [dict(obs=torch.tensor(p['obs'], dtype=dt), act=torch.tensor(p['act'], dtype=dt),
                 adv=torch.tensor(p['adv'], dtype=dt), mean=torch.tensor(p['mean'], dtype=dt),
                 log_std=torch.tensor(p['log_std'], dtype=dt)[:, None, :].expand(-1, N, -1),
                 adj_avg_rewards=torch.tensor(p['adj_avg_rewards'], dtype=dt)) for p in case['phases']]


@pytest.mark.parametrize('act,name', GOLDEN_CASES, ids=GOLDEN_IDS)
def test_otanh_oracle_matches_reference_graph(golden_dir, act, name, otanh_oracle):
    """The float64 tanh-output oracle == the unmodified reference graph with output_nonlinearity=tf.tanh, evaluated in
    float64: adapted parameters, objective, KLs, second-order meta-gradient, and for TRPO-MAML the KL gradient and the
    Hessian-vector product of the KL."""
    _use(otanh_oracle, act)
    G = _gold(golden_dir)
    case = tf_cases.make_case(name)
    dt, tol = torch.float64, 1e-6
    lr = float(np.float32(0.1))         # the reference's inner_lr is a float32 constant
    pre = '%s/%s/f64/' % (name, act)
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


@pytest.mark.parametrize('kind', ['ratio', 'loglik'])
def test_otanh_hvp_oracle_matches_central_differences(kind):
    """The exact HVP (double backward through the tanh-output oracle, with its second-order term of the output layer) ==
    central differences of its gradient."""
    case = po.Case(5, 3, 32, 3, 200, seed=21)
    vec = case.vec()
    want = case.hvp_delta(kind, vec, 1.0, 0.0).numpy()
    fd = po._central_difference_hvp(case, kind, vec).numpy()
    po.assert_blocks('central differences ' + kind, fd, want, 5, 3, 32)


def test_otanh_and_identity_oracles_differ(otanh_oracle):
    """The same weights with a tanh and an identity output layer give gradients and HVPs far apart (outside the bar), with
    either hidden activation: a kernel that ignored the flag fails the GPU tests."""
    for act, identity in (('tanh', IDENTITY_DIST_INFO), ('relu', None)):
        case = po.Case(2, 2, 32, 2, 100, seed=3)
        vec = case.vec()
        _use(otanh_oracle, act)
        otanh = case.grad('ratio')[0].numpy(), case.hvp_delta('ratio', vec, 0.1, 0.0).numpy()
        if identity is None:        # ReLU hidden layers, identity output (the forward of test_relu_policy.py)
            def identity(theta, obs, dims, min_log_std=None):
                W0, b0, W1, b1, W2, b2, ls = th.split_params(theta, *dims)
                h = torch.relu(torch.relu(torch.matmul(obs, W0) + b0.unsqueeze(-2)) @ W1 + b1.unsqueeze(-2))
                return torch.matmul(h, W2) + b2.unsqueeze(-2), (ls if min_log_std is None else torch.clamp(ls, min=min_log_std))
        otanh_oracle.setattr(th, 'dist_info', identity)
        ident = case.grad('ratio')[0].numpy(), case.hvp_delta('ratio', vec, 0.1, 0.0).numpy()
        assert not po.blocks_pass(otanh[0], ident[0], 2, 2, 32) and not po.blocks_pass(otanh[1], ident[1], 2, 2, 32), act


def _shim_tf():
    import importlib.util
    shim = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'promp_b200', 'tf_shim', 'tensorflow',
                        '__init__.py')
    spec = importlib.util.spec_from_file_location('promp_tf_shim', shim)      # not as `tensorflow`: oracle/stubs_tf owns that name
    tf = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tf)
    return tf


def test_output_activation_names():
    """output_nonlinearity accepted by MetaGaussianMLPPolicy: None (identity), 'tanh', or a callable named tanh (the tf_shim
    placeholder that run scripts pass, torch.tanh); every other value is unsupported."""
    from promp_b200.policies.meta_gaussian_mlp_policy import _output_activation_name
    tf = _shim_tf()
    assert _output_activation_name(None) is None
    for fn in ('tanh', tf.tanh, torch.tanh):
        assert _output_activation_name(fn) == 'tanh', fn
    for fn in (tf.nn.relu, torch.sigmoid, 'sigmoid', lambda x: x, 'Tanh', 3):
        assert _output_activation_name(fn) is False, fn


def test_abi_out_tanh_flag():
    """PROMP_OUT_TANH in the `hidden` argument, alone and with PROMP_ACT_RELU: num_params / layout / workspace sizes unchanged;
    unknown bits and the flag at an unsupported width rejected (before any device work: these calls are safe without a
    GPU)."""
    import ctypes
    from promp_b200 import _lib
    lib = _lib.load()
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'promp_b200.h')).read()
    assert '#define PROMP_OUT_TANH 0x%x' % _lib.OUT_TANH in header
    O, R = _lib.OUT_TANH, _lib.ACT_RELU
    for Do, Da in ((2, 2), (17, 6), (5, 3), (19, 8)):
        for h in (32, 64):
            for flags in (O, O | R):
                assert lib.promp_num_params(Do, Da, h | flags) == lib.promp_num_params(Do, Da, h) == th.num_params(Do, Da, (h, h))
                assert _lib.policy_layout(Do, Da, h | flags) == _lib.policy_layout(Do, Da, h)
                assert (lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h | flags)
                        == lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h))
                assert (lib.promp_policy_workspace_bytes_padded(40, 2000, Do, Da, h | flags)
                        == lib.promp_policy_workspace_bytes_padded(40, 2000, Do, Da, h))
    for bits in (0x200, 0x400, 0x800, 0x2000):
        with pytest.raises(_lib.PrompLibraryError, match='unknown flag bits'):
            _lib.policy_layout(2, 2, 64 | O | bits)
    for flags in (O, O | R):
        with pytest.raises(_lib.PrompLibraryError, match='built for hidden 32 or 64'):
            _lib.policy_layout(2, 2, 48 | flags)
    with pytest.raises(_lib.PrompLibraryError, match='tanh-output policies are built for hidden 32 or 64'):
        _lib.policy_layout(2, 2, 16 | O)
    dummy = 16
    for hidden, msg in ((64 | O | 0x400, 'unknown flag bits'), (16 | O, 'tanh-output policies are built for hidden 32 or 64'),
                        (128 | O, 'tanh-output policies are built for hidden 32 or 64')):
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
    stage = _lib.PolicyStage(kind=0, N=100)          # read on the host only
    for fn in (lib.promp_policy_chain_workspace_bytes, lib.promp_policy_chain_num_launches):
        for flags in (O, O | R):
            assert fn(2, 2, 64 | flags, 4, 1, ctypes.byref(stage)) == fn(2, 2, 64, 4, 1, ctypes.byref(stage)) > 0
        assert fn(2, 2, 64 | O | 0x200, 4, 1, ctypes.byref(stage)) == -1


# ================================================================================================================ GPU
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from promp_b200 import _lib
    _lib.require_cuda()


def _otanh_policy(Do, Da, hidden_sizes, M, act='tanh', output='tanh'):
    from promp_b200.policies import MetaGaussianMLPPolicy
    return MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=hidden_sizes,
                                 hidden_nonlinearity=act, output_nonlinearity=output)


class OtanhLauncher(po.Launcher):
    """test_policy_oracle.Launcher on a tanh-output policy: every call passes `policy.hidden_arg`."""

    def __init__(self, case, act='tanh'):
        orig = po._policy
        po._policy = lambda c: _otanh_policy(c.Do, c.Da, (c.hidden, c.hidden), c.M, act)
        try:
            super(OtanhLauncher, self).__init__(case)
        finally:
            po._policy = orig
        from promp_b200 import _lib
        assert self.pol.hidden_arg == self.pol.hidden | _lib.OUT_TANH | (_lib.ACT_RELU if act == 'relu' else 0)

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


def _otanh_kernels(path, Do, Da, hidden):
    """The path's kernel names with the tanh output: policy_*_otanh_kernel<shape..., hidden activation>."""
    return [k.replace('_kernel<', '_otanh_kernel<')[:-1] + ',' for k in po._expected_kernels(path, Do, Da, hidden)]


SHAPES = po.EXACT_SHAPES + po.BUCKET_SHAPES


@pytest.mark.gpu
@pytest.mark.parametrize('act', ['tanh', 'relu'])
@pytest.mark.parametrize('Do,Da', SHAPES, ids=['%dx%d' % s for s in SHAPES])
@pytest.mark.parametrize('path', po.PATHS)
def test_otanh_kernels_match_oracle(path, Do, Da, act, otanh_oracle):
    """Gradient (RATIO + KL, CLIP), HVP (RATIO, LOGLIK) and forward of every kernel path at every exact and bucket shape,
    with tanh and ReLU hidden layers, against the float64 tanh-output oracle; N = 300 fills no 64- or 128-sample tile
    exactly; the kernels the profiler records are the path's tanh-output kernels."""
    _cuda()
    _use(otanh_oracle, act)
    hidden = 32 if path == 'h32' else 64
    case = po.Case(Do, Da, hidden, 3, 300, seed=300 + Do * 10 + Da)
    with po._path(path):
        L = OtanhLauncher(case, act)
        what = 'otanh %s %s %dx%d' % (act, path, Do, Da)
        po.check_grad(L, what, 'ratio', kl_coeff=0.1)
        po.check_grad(L, what, 'clip', kl_coeff=0.2)
        po.check_hvp(L, what, 'ratio')
        po.check_hvp(L, what, 'loglik')
        mu, _ = DIST[act](case.theta_t(), case.data()['obs'], case.dims)
        np.testing.assert_allclose(L.forward(), mu.numpy(), rtol=1e-4, atol=1e-5)
        names = po._kernels_run_by(lambda: (L.grad('ratio'), L.hvp('ratio', case.vec())))
    expected = _otanh_kernels(path, Do, Da, hidden)
    for k in set(k for k in (names or []) if 'policy_' in k):
        assert any(name in k for name in expected), (k, expected)
        assert ('ActRelu' in k) == (act == 'relu'), k


@pytest.mark.gpu
@pytest.mark.parametrize('act', ['tanh', 'relu'])
@pytest.mark.parametrize('path', ['cuda', 'tc512', 'h32'])
def test_otanh_ragged_shared_and_deterministic(path, act, otanh_oracle):
    """Ragged n_valid with poisoned padding, shared parameters with a binding log_std clip, per-sample old log_std; two
    launches give the same bits."""
    _cuda()
    _use(otanh_oracle, act)
    hidden = 32 if path == 'h32' else 64
    M = 4
    cases = [po.Case(2, 2, hidden, M, 257, seed=7, n_valid=[257, 1, 130, 64]),
             po.Case(17, 6, hidden, M, 200, seed=8, shared=True, ls=po._binding_ls(1, 6, -0.3, 9), min_log_std=-0.3),
             po.Case(5, 3, hidden, M, 129, seed=9, ls_per_sample=True)]
    with po._path(path):
        for case in cases:
            L = OtanhLauncher(case, act)
            what = 'otanh %s %s %dx%d' % (act, path, case.Do, case.Da)
            po.check_grad(L, what, 'ratio', kl_coeff=0.1)
            po.check_hvp(L, what, 'ratio')
            g1, _, s1 = L.grad('clip', kl_coeff=0.1)
            g2, _, s2 = L.grad('clip', kl_coeff=0.1)
            vec = case.vec()
            _, o1, _ = L.hvp('ratio', vec)
            _, o2, _ = L.hvp('ratio', vec)
            assert torch.equal(g1, g2) and torch.equal(s1[:, :3], s2[:, :3]) and torch.equal(o1, o2), what


@pytest.mark.gpu
def test_otanh_saturated_mean():
    """Large output pre-activations (|z| up to ~10) drive the mean into tanh's saturation, where 1 - mu^2 underflows
    towards 0: the gradient and HVP still meet the bar, on CUDA and tensor cores."""
    _cuda()
    case = po.Case(2, 2, 64, 3, 300, seed=77)
    th_l = case.theta_tasks.copy()
    dims = case.dims
    P = th.num_params(*dims)
    th_l[:, P - 2 * 2 - 64 * 2:P - 2 * 2] *= 6.0          # W2 and b2 of the (2, 2) policy
    case.theta_tasks = th_l.astype(np.float32)
    mu, _ = DIST['tanh'](case.theta_t(), case.data()['obs'], dims)
    assert float((mu.abs() > 0.999).double().mean()) > 0.05
    for path in ('cuda', 'tc512'):
        with po._path(path):
            L = OtanhLauncher(case)
            po.check_grad(L, 'saturated ' + path, 'ratio', kl_coeff=0.1)
            po.check_hvp(L, 'saturated ' + path, 'ratio')


def _product_algo(case, act, **kw):
    from promp_b200.meta_algos import ProMP, TRPOMAML, VPGMAML
    H = tf_cases.HYPER
    M, S1 = case['M'], case['S'] - 1
    np.random.seed(1)
    policy = _otanh_policy(case['Do'], case['Da'], (case['hidden'],) * 2, M, act)
    policy.set_params(tf_cases.unflatten(case['theta'], case['Do'], case['Da'], case['hidden']))
    if case['algo'] == 'promp':
        algo = ProMP(policy=policy, inner_lr=H['inner_lr'], meta_batch_size=M, num_inner_grad_steps=S1,
                     learning_rate=H['learning_rate'], num_ppo_steps=H['num_ppo_steps'], clip_eps=H['clip_eps'],
                     target_inner_step=0.01, init_inner_kl_penalty=H['init_inner_kl_penalty'], adaptive_inner_kl_penalty=False)
    elif case['algo'] == 'trpo':
        algo = TRPOMAML(policy=policy, step_size=H['step_size'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                        meta_batch_size=M, num_inner_grad_steps=S1, **kw)
    else:
        algo = VPGMAML(policy=policy, learning_rate=H['learning_rate'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                       meta_batch_size=M, num_inner_grad_steps=S1, **kw)
    return policy, algo


@pytest.mark.gpu
@pytest.mark.parametrize('act,name', GOLDEN_CASES, ids=GOLDEN_IDS)
def test_otanh_adapt_and_meta_gradient_match_reference_graph(golden_dir, act, name):
    """MAMLAlgo._adapt (SGD) and the second-order meta-gradient of a tanh-output policy on the device against the unmodified
    reference graph with output_nonlinearity=tf.tanh (float64 evaluation), at the 1e-4 bar.  ProMP / VPG-MAML: the dataflow
    chain and one launch per stage give the same gradient."""
    _cuda()
    from promp_b200 import _lib
    G = _gold(golden_dir)
    case = tf_cases.make_case(name)
    samples = tf_cases.reference_samples(case)
    pre = '%s/%s/f64/' % (name, act)
    th0 = case['theta'].astype(np.float64)
    grads = {}
    for chain in ((1, 0) if case['algo'] != 'trpo' else (-1,)):
        _lib.set_option('chain', chain)
        try:
            policy, algo = _product_algo(case, act)
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


@pytest.mark.gpu
@pytest.mark.parametrize('act', ['tanh', 'relu'])
@pytest.mark.parametrize('ragged', [False, True])
def test_otanh_chain_with_exploration_matches_per_stage_launches(ragged, act, otanh_oracle):
    """The E-MAML meta-gradient (inner step, outer gradient, HVP, exploration stage) of a tanh-output policy: the dataflow
    chain equals one launch per stage (same sums up to order) and repeats bit for bit, on fixed-length and ragged phases."""
    _cuda()
    _use(otanh_oracle, act)
    import test_emaml as em
    from promp_b200 import _lib
    M, Do, Da, N = 6, 2, 2, 700
    np.random.seed(1)
    policy = _otanh_policy(Do, Da, (64, 64), M, act)
    th_l = policy.unpad_flat(policy.theta.cpu().numpy()).copy()
    th_l += 0.1 * np.random.RandomState(9).randn(th_l.size).astype(np.float32)
    policy.set_params(th_l)
    algo = em._trpo(policy, M)
    if ragged:
        lens = [[120, 300, 200], [620], [1, 5, 400], [250, 250], [90], [700]]
        phases = [em._ragged_phase(torch, lens, Do, Da, th_l, 40 + s)[1] for s in range(2)]
    else:
        phases = [em._fixed_phase(torch, M, N, Do, Da, th_l, 30 + s)[1] for s in range(2)]
    c = algo.exploration_coeff_dev(phases)

    def run(mode):
        algo.use_chain = True
        _lib.set_option('chain', 1 if mode == 'dataflow' else 0)
        try:
            res = algo._meta_pass(policy.theta, phases, _lib.OBJ_RATIO, 0.0, [0.0], want_grad=True, explore=c)
            torch.cuda.synchronize()
        finally:
            _lib.set_option('chain', -1)
        return res['grad'].clone(), res['explore'].clone()
    g0, x0 = run('per_stage')
    g1, x1 = run('dataflow')
    g2, x2 = run('dataflow')
    assert torch.isfinite(g0).all() and torch.equal(g1, g2) and torch.equal(x1, x2)
    assert rel_err(g1.cpu().numpy(), g0.cpu().numpy()) < 2e-5, rel_err(g1.cpu().numpy(), g0.cpu().numpy())
    np.testing.assert_allclose(x1.cpu().numpy(), x0.cpu().numpy(), rtol=2e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------ fused rollout
# (env kind, obs, act, task floats, early-terminating)
ROLLOUT_ENVS = dict(point_corner=(0, 2, 2, 2, False), point=(1, 2, 2, 1, True), cheetah=(2, 17, 6, 1, False),
                    swimmer=(6, 8, 2, 1, False), walker=(5, 17, 6, 2, True))


def _rollout(kind, early, M, E, T, H, hidden_arg, params, PL, task_d, noise_d, obs, act, mean, rew, done, info, ls_out):
    from promp_b200 import _lib
    p = _lib.ptr
    if early:
        _lib.call('promp_rollout_early_term', kind, 1, M, E, T, H, hidden_arg, p(params), PL, p(task_d), None, p(noise_d),
                  5, 1, None, 0, -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(ls_out), _lib.stream())
    else:
        _lib.call('promp_rollout', kind, 0 if kind != 0 else 1, 0.5, 1, M, E, H, hidden_arg, p(params), PL, p(task_d), None,
                  p(noise_d), 5, 1, None, 0, -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(info), p(ls_out), None,
                  _lib.stream())
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('act', ['tanh', 'relu'])
@pytest.mark.parametrize('hidden', [64, 32])
@pytest.mark.parametrize('env', list(ROLLOUT_ENVS))
def test_otanh_fused_rollout_teacher_forced(env, hidden, act):
    """promp_rollout (fixed horizon) / promp_rollout_early_term (device resets) with a tanh-output policy and fed noise: the
    recorded means against the float64 tanh-output policy evaluated on the kernel's own observations, and
    act = mean + eps * exp(log_std); the identity-output kernel records different means on the same inputs."""
    _cuda()
    from promp_b200 import _lib
    kind, Do, Da, TD, early = ROLLOUT_ENVS[env]
    M, E, H = 3, 6, 40
    rng = np.random.RandomState(kind * 10 + hidden + (1 if act == 'relu' else 0))
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
    obs, a_d, mean = (torch.empty(M, E, T, n, device='cuda') for n in (Do, Da, Da))
    rew = torch.empty(M, E, T, device='cuda')
    done = torch.empty(M, E, T, dtype=torch.uint8, device='cuda')
    ls_out = torch.empty(M, Da, device='cuda')
    info = torch.zeros(3, M, E, T, device='cuda')
    base = hidden | (_lib.ACT_RELU if act == 'relu' else 0)
    params, task_d, noise_d = dev(theta), dev(task), dev(noise)
    bufs = (obs, a_d, mean, rew, done, info, ls_out)
    _rollout(kind, early, M, E, T, H, base | _lib.OUT_TANH, params, PL, task_d, noise_d, *bufs)
    o, a, mu = obs.cpu().numpy(), a_d.cpu().numpy(), mean.cpu().numpy()
    if early:
        assert done.cpu().numpy().sum() >= M * E        # every slot finished at least one path and kept stepping after its reset
    assert np.abs(mu).max() < 1.0
    want, _ = DIST[act](torch.from_numpy(theta).double(), torch.from_numpy(o.reshape(M, E * T, Do)).double(), dims)
    want = want.numpy().reshape(M, E, T, Da)
    np.testing.assert_allclose(mu, want, rtol=1e-4, atol=2e-5)
    sig = np.exp(theta[:, -Da:].astype(np.float64))[:, None, None, :]
    np.testing.assert_allclose(a, mu + noise * sig, rtol=1e-5, atol=1e-5)
    _rollout(kind, early, M, E, T, H, base, params, PL, task_d, noise_d, *bufs)
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
    if kind in ('point', 'emaml'):
        env = normalize(MetaPointEnvCorner(reward_type='dense'))    # sparse rewards give all-zero advantages at this size
    elif kind == 'cheetah':
        env = normalize(HalfCheetahRandDirecEnv())
    else:
        env = normalize(Walker2DRandVelEnv())
        sampler_kw = dict(reset_mode='device')
    Do, Da = int(np.prod(env.observation_space.shape)), int(np.prod(env.action_space.shape))
    policy = _otanh_policy(Do, Da, (64, 64), M, output=torch.tanh)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H, **sampler_kw)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    if kind == 'emaml':
        algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, step_size=0.01, exploration=True)
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
@pytest.mark.parametrize('kind,graph', [('point', True), ('cheetah', True), ('emaml', False), ('walker', False)])
def test_otanh_trainer_runs(kind, graph, tmp_path):
    """Three meta-iterations of Trainer.train() with a tanh-output policy: ProMP in CUDA-graph mode (point, cheetah),
    TRPO-MAML with exploration=True, and the walker with device resets (early termination).  Every logged scalar is finite
    and the same seed gives the same results; the snapshot keeps the output activation."""
    _cuda()
    policy, kv = _train(kind, tmp_path / 'a', seed=11, graph=graph)
    policy2, kv2 = _train(kind, tmp_path / 'b', seed=11, graph=graph)
    assert kv['Itr'] == 2
    for key in ('Step_0-AverageReturn', 'Step_1-AverageReturn'):
        assert key in kv, key
    assert all(np.isfinite(v) for k, v in kv.items() if isinstance(v, (float, int, np.floating)) and 'Time' not in k)
    assert torch.equal(policy.theta, policy2.theta)
    for k, v in kv.items():
        if 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert v == kv2[k], k
    from promp_b200.utils import logger
    snap = logger.load_snapshot(os.path.join(str(tmp_path / 'a'), 'params.pkl'))
    pol = snap['policy']
    assert pol.output_nonlinearity == 'tanh' and pol.hidden_arg == policy.hidden_arg
    assert torch.equal(pol.theta, policy.theta)


@pytest.mark.gpu
def test_otanh_policy_constructor_pickle_and_get_actions():
    _cuda()
    from promp_b200 import _lib
    from promp_b200.policies import MetaGaussianMLPPolicy
    tf = _shim_tf()
    for out in ('tanh', tf.tanh, torch.tanh):
        pol = _otanh_policy(2, 2, (32, 32), 2, output=out)
        assert pol.output_nonlinearity == 'tanh' and pol.hidden_arg == 32 | _lib.OUT_TANH
    assert _otanh_policy(2, 2, (32, 32), 2, act='relu').hidden_arg == 32 | _lib.ACT_RELU | _lib.OUT_TANH
    ident = _otanh_policy(2, 2, (32, 32), 2, output=None)
    assert ident.output_nonlinearity is None and ident.hidden_arg == 32
    for bad in (tf.nn.relu, torch.sigmoid, lambda x: x):
        with pytest.raises(NotImplementedError, match='identity or tanh output'):
            _otanh_policy(2, 2, (32, 32), 2, output=bad)
    pol = _otanh_policy(17, 6, (64, 64), 3, act='relu')
    pol2 = pickle.loads(pickle.dumps(pol))
    assert pol2.output_nonlinearity == 'tanh' and pol2.hidden_arg == pol.hidden_arg and torch.equal(pol2.theta, pol.theta)
    # a state saved before the output activation was stored loads with the identity output
    state = pol.__getstate__()
    del state['init_args']['output_nonlinearity']
    old = MetaGaussianMLPPolicy.__new__(MetaGaussianMLPPolicy)
    old.__setstate__(state)
    assert old.output_nonlinearity is None and old.hidden_arg == 64 | _lib.ACT_RELU
    # get_actions (promp_policy_forward) with the tanh output, exact and padded shapes
    for p_, (Do, Da) in ((pol, (17, 6)), (_otanh_policy(5, 3, (64, 64), 3), (5, 3))):
        obs = [np.random.RandomState(m).randn(5, Do).astype(np.float32) for m in range(3)]
        _, infos = p_.get_actions(obs)
        theta = torch.from_numpy(p_.unpad_flat(p_.theta.cpu().numpy())).double()[None].expand(3, -1)
        want, _ = DIST[p_.hidden_nonlinearity](theta, torch.from_numpy(np.stack(obs)).double(), (Do, Da, (64, 64)))
        got = np.stack([[infos[m][e]['mean'] for e in range(5)] for m in range(3)])
        np.testing.assert_allclose(got, want.numpy(), rtol=1e-4, atol=1e-5)
