"""Policies with one or three hidden layers (hidden_sizes of length 1 to 3): the depth field of the `hidden` argument, the
parameter layout of every depth, and the CUDA-core kernels of depth 1 and 3 (gradient, Hessian-vector product, forward,
fused rollout, chain) against a float64 autograd statement of the reference's policy.

The float64 policy below is forward_mlp (policies/networks/mlp.py:65-119) for any number of hidden layers, with the
distribution functions pinned in oracle/tf_half.py (log_likelihood, likelihood_ratio, kl).  Results are compared per task
and per parameter block (every kernel and bias of the mean network, then log_std) at the bar of test_policy_oracle.py:
    |got - want|_mb <= RTOL |want_mb| + FLOOR |want_m|.

CPU: layout, decoding and rejection of the depth bits, two-layer values unchanged, the JIT's kernel names.
GPU (-m gpu): the kernels, get_actions, the fused rollouts (built-in and user envs), the chain and Trainer.train().
"""
import contextlib
import math
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import tf_half as th

RTOL, FLOOR = 1e-4, 2e-5            # test_policy_oracle.py
MIN_LOG_STD = math.log(1e-6)
CLIP_EPS = 0.3
OBJ = dict(ratio=0, loglik=1, clip=2, explore=4)
EXACT_SHAPES = ((2, 2), (4, 2), (17, 6))


def _caps(Do, Da):
    if (Do, Da) in EXACT_SHAPES:
        return Do, Da
    return (8 if Do <= 8 else 20), (2 if Da <= 2 else 8)


# ------------------------------------------------------------------------------------------------------ float64 policy
def ref_shapes(Do, Da, sizes):
    """The reference's variables in creation order (create_mlp: hidden_i kernel / bias, output kernel / bias; then log_std)."""
    ins = (Do,) + tuple(sizes)
    out = []
    for i in range(len(sizes)):
        out += [('mean_network/hidden_%d/kernel' % i, (ins[i], ins[i + 1])), ('mean_network/hidden_%d/bias' % i, (ins[i + 1],))]
    return out + [('mean_network/output/kernel', (sizes[-1], Da)), ('mean_network/output/bias', (Da,)),
                  ('log_std_network/log_std_var', (1, Da))]


def n_logical(Do, Da, sizes):
    return sum(int(np.prod(s)) for _, s in ref_shapes(Do, Da, sizes))


def split(theta, Do, Da, sizes):
    out, off = [], 0
    lead = theta.shape[:-1]
    for _, shape in ref_shapes(Do, Da, sizes):
        n = int(np.prod(shape))
        out.append(theta[..., off:off + n].reshape(*lead, *shape))
        off += n
    return out


def dist_info(theta, obs, dims, act='tanh', out=None):
    """theta [M,P], obs [M,N,Do] -> mean [M,N,Da], log_std [M,1,Da]"""
    Do, Da, sizes = dims
    p = split(theta, Do, Da, sizes)
    f = torch.tanh if act == 'tanh' else torch.relu
    h = obs
    for i in range(len(sizes)):
        h = f(torch.matmul(h, p[2 * i]) + p[2 * i + 1].unsqueeze(-2))
    mean = torch.matmul(h, p[-3]) + p[-2].unsqueeze(-2)
    if out == 'tanh':
        mean = torch.tanh(mean)
    return mean, p[-1]


def terms(theta, d, dims, kind, act, out, min_log_std=None):
    mean, ls = dist_info(theta, d['obs'], dims, act, out)
    if min_log_std is not None:
        ls = torch.clamp(ls, min=min_log_std)
    ratio = th.likelihood_ratio(d['act'], d['mean'], d['log_std'], mean, ls)
    if kind == 'ratio':
        per = ratio * d['adv']
    elif kind == 'clip':
        per = torch.minimum(ratio * d['adv'], torch.clamp(ratio, 1 - CLIP_EPS, 1 + CLIP_EPS) * d['adv'])
    else:       # loglik; explore = loglik with the per-task weight broadcast over the samples
        per = th.log_likelihood(d['act'], mean, ls) * d['adv']
    kl = torch.mean(th.kl(d['mean'], d['log_std'], mean, ls), -1)
    return -torch.mean(per, -1), kl, torch.mean(ratio, -1)


def oracle_grad(theta, d, dims, kind, act, out, kl_coeff=0.0, min_log_std=None):
    t = theta.detach().clone().requires_grad_(True)
    surr, kl, ratio = terms(t, d, dims, kind, act, out, min_log_std)
    (g,) = torch.autograd.grad((surr + kl_coeff * kl).sum(), t)
    return g, torch.stack([surr, kl, ratio], -1).detach()


def oracle_hvp_delta(theta, d, dims, kind, act, out, vec, inner_lr, kl_coeff, min_log_std=None):
    t = theta.detach().clone().requires_grad_(True)
    surr, kl, _ = terms(t, d, dims, kind, act, out, min_log_std)
    (g,) = torch.autograd.grad(surr.sum(), t, create_graph=True)
    (hv,) = torch.autograd.grad((g * vec).sum(), t, retain_graph=True)
    (gk,) = torch.autograd.grad(kl.sum(), t)
    return -inner_lr * hv + kl_coeff * gk


def block_ratios(got, want, dims):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    norm_m = np.linalg.norm(want, axis=1)
    shapes = ref_shapes(*dims)
    out, off = np.zeros((want.shape[0], len(shapes))), 0
    for b, (_, shape) in enumerate(shapes):
        sl = slice(off, off + int(np.prod(shape)))
        off = sl.stop
        err = np.linalg.norm(got[:, sl] - want[:, sl], axis=1)
        bound = RTOL * np.linalg.norm(want[:, sl], axis=1) + FLOOR * norm_m
        with np.errstate(divide='ignore', invalid='ignore'):
            out[:, b] = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return out


def assert_blocks(what, got, want, dims):
    r = block_ratios(got, want, dims)
    if not np.all(r <= 1.0):
        m, b = np.unravel_index(np.argmax(r), r.shape)
        raise AssertionError('%s: task %d block %s at %.2fx the bound (%d pairs over)'
                             % (what, m, ref_shapes(*dims)[b][0], r[m, b], int((r > 1).sum())))


# ------------------------------------------------------------------------------------------------------------ CPU
def _bits(depth):
    from promp_b200 import _lib
    return _lib.hidden_depth(depth)


def test_header_depth_field_mirrors_lib():
    from promp_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'promp_b200.h')).read()
    assert '#define PROMP_HIDDEN_DEPTH_SHIFT %d' % _lib.HIDDEN_DEPTH_SHIFT in header
    assert '#define PROMP_HIDDEN_DEPTH_MASK 0x%X' % _lib.HIDDEN_DEPTH_MASK in header
    assert '#define PROMP_ENV_MODULE_SLOTS %d' % _lib.ENV_MODULE_SLOTS in header
    assert '#define PROMP_ENV_SLOT_ROLLOUT_DEEP %d' % _lib.ENV_SLOT_ROLLOUT_DEEP in header
    assert _lib.hidden_depth(2) == 0 and _lib.hidden_depth(1) == 0x4000 and _lib.hidden_depth(3) == 0xC000
    # bits the other flags' tests keep unknown stay outside the field
    for bits in (0x200, 0x400, 0x800, 0x2000):
        assert bits & _lib.HIDDEN_DEPTH_MASK == 0


@pytest.mark.parametrize('depth', [1, 2, 3])
@pytest.mark.parametrize('hidden', [32, 64])
@pytest.mark.parametrize('Do,Da', [(2, 2), (4, 2), (17, 6), (1, 1), (5, 3), (8, 2), (19, 8)])
def test_num_params_and_layout_match_reference_variables(Do, Da, hidden, depth):
    """promp_num_params / promp_policy_layout with the depth bits = the sizes of the variables the reference creates for
    hidden_sizes = (hidden,) * depth at the zero-padded caps, with any activation flags."""
    from promp_b200 import _lib
    lib = _lib.load()
    cd, ca = _caps(Do, Da)
    want = n_logical(cd, ca, (hidden,) * depth)
    for flags in (0, _lib.ACT_RELU, _lib.OUT_TANH, _lib.ACT_RELU | _lib.OUT_TANH):
        h = hidden | flags | _bits(depth)
        assert lib.promp_num_params(cd, ca, h) == want
        lay = _lib.policy_layout(Do, Da, h)
        assert lay[:3] == ((8 if Do <= 8 else 20), (2 if Da <= 2 else 8), hidden)
        assert lay[3] == n_logical(lay[0], lay[1], (hidden,) * depth) and lay[3] % 4 == 0


def test_two_layers_keep_every_value():
    """No depth bits = two hidden layers: num_params, the layout and every workspace size are what they were, and the
    explicit depth-2 field means the same."""
    from promp_b200 import _lib
    lib = _lib.load()
    D2 = 2 << _lib.HIDDEN_DEPTH_SHIFT
    for Do, Da in ((2, 2), (17, 6), (5, 3), (19, 8)):
        for h in (32, 64):
            P = lib.promp_num_params(Do, Da, h)
            assert P == th.num_params(Do, Da, (h, h)) == lib.promp_num_params(Do, Da, h | D2)
            assert _lib.policy_layout(Do, Da, h | D2) == _lib.policy_layout(Do, Da, h)
            assert lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h | D2) == lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h)
    assert lib.promp_num_params(2, 2, 64) == 4484 and lib.promp_num_params(17, 6, 64) == 5708


def test_deep_workspace_and_chain_queries():
    """The workspace grows with P; the chain of a deep policy runs its stages as one launch each and its workspace holds
    the largest stand-alone launch after the control words (host-only queries)."""
    import ctypes
    from promp_b200 import _lib
    lib = _lib.load()
    stages = (_lib.PolicyStage * 3)(_lib.PolicyStage(kind=0, N=2000), _lib.PolicyStage(kind=0, N=2000),
                                    _lib.PolicyStage(kind=1, N=2000))
    sp = ctypes.cast(stages, ctypes.c_void_p)
    for Do, Da in ((2, 2), (17, 6)):
        w = [lib.promp_policy_workspace_bytes(40, 2000, Do, Da, 64 | _bits(d)) for d in (1, 2, 3)]
        assert w[0] < w[1] < w[2]
        for d in (1, 3):
            h = 64 | _bits(d)
            assert lib.promp_policy_chain_num_launches(Do, Da, h, 40, 3, sp) == 3
            ws = lib.promp_policy_chain_workspace_bytes(Do, Da, h, 40, 3, sp)
            assert ws > lib.promp_policy_workspace_bytes(40, 2000, Do, Da, h)
    assert lib.promp_policy_chain_num_launches_padded(5, 3, 32 | _bits(3), 40, 3, sp) == 3
    assert (lib.promp_policy_chain_workspace_bytes_padded(5, 3, 32 | _bits(1), 40, 3, sp)
            > lib.promp_policy_workspace_bytes_padded(40, 2000, 5, 3, 32 | _bits(1)))


def test_depth_bits_rejected_outside_their_range():
    """Field values 4..7 (more than three hidden layers) and the depth field at a width other than 32 / 64 are rejected by
    every entry point before any device work (safe without a GPU)."""
    from promp_b200 import _lib
    lib = _lib.load()
    for field in (4, 5, 6, 7):
        with pytest.raises(_lib.PrompLibraryError, match='1 to 3 hidden layers'):
            _lib.policy_layout(2, 2, 64 | (field << _lib.HIDDEN_DEPTH_SHIFT))
    for width in (48, 16, 128):
        with pytest.raises(_lib.PrompLibraryError, match='depth 1 or 3 are built for hidden 32 or 64'):
            _lib.policy_layout(2, 2, width | _bits(3))
    with pytest.raises(_lib.PrompLibraryError, match='unknown flag bits'):
        _lib.policy_layout(2, 2, 64 | _bits(3) | 0x2000)
    dummy = 16
    for hidden, msg in ((64 | (4 << _lib.HIDDEN_DEPTH_SHIFT), '1 to 3 hidden layers'),
                        (48 | _bits(1), 'depth 1 or 3 are built for hidden 32 or 64')):
        assert lib.promp_policy_forward(2, 2, hidden, 1, 1, dummy, 0, dummy, dummy, None) == -1
        assert msg in _lib.last_error()
        assert lib.promp_rollout(_lib.ENV_POINT_CORNER, 0, 0.5, 1, 1, 1, 4, hidden, dummy, 0, dummy, None, None, 1, 1, None, 1,
                                 -13.8, dummy, dummy, dummy, dummy, dummy, None, dummy, None, None) == -1
        assert msg in _lib.last_error()
        assert lib.promp_rollout_early_term(_lib.ENV_POINT, 1, 1, 1, 8, 4, hidden, dummy, 0, dummy, None, None, 1, 1, None, 1,
                                            -13.8, dummy, dummy, dummy, dummy, dummy, dummy, None) == -1
        assert msg in _lib.last_error()
    assert lib.promp_num_params(2, 2, 64 | (4 << _lib.HIDDEN_DEPTH_SHIFT)) == -1


def test_jit_names_the_deep_rollout_kernel():
    from promp_b200 import _jit, _lib
    for h in (64, 32 | _lib.ACT_RELU, 64 | _lib.OUT_TANH):
        assert _jit.rollout_slot(h, False) < _lib.ENV_SLOT_ROLLOUT_DEEP
        for d in (1, 3):
            hd = h | _bits(d)
            slot = _jit.rollout_slot(hd, True)
            assert slot == _jit.rollout_slot(h, True) - _lib.ENV_SLOT_ROLLOUT + _lib.ENV_SLOT_ROLLOUT_DEEP
            assert slot < _lib.ENV_MODULE_SLOTS
            names = _jit.name_expressions([hd])
            assert names[slot].startswith('promp::rollout_deep_kernel<promp_jit::Env, %d, ' % (h & 0xFF))
            assert names[slot].endswith(', true>')
    with pytest.raises(ValueError):
        _jit.rollout_slot(64 | (5 << _lib.HIDDEN_DEPTH_SHIFT), False)


def test_float64_policy_is_the_two_layer_oracle_at_depth_two():
    """The depth-generic float64 policy used by the GPU tests equals oracle/tf_half.dist_info for two tanh layers."""
    rng = np.random.RandomState(0)
    dims = (5, 3, (64, 64))
    theta = torch.from_numpy(th.init_params(*dims, rng=rng).astype(np.float64)[None] + 0.1 * rng.randn(2, th.num_params(*dims)))
    obs = torch.from_numpy(rng.randn(2, 7, 5))
    a, _ = dist_info(theta, obs, dims)
    b, _ = th.dist_info(theta, obs, dims)
    assert torch.allclose(a, b, rtol=0, atol=1e-14)
    assert [s for _, s in ref_shapes(*dims)] == list(th.param_shapes(*dims).values())


# ------------------------------------------------------------------------------------------------------------ GPU
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from promp_b200 import _lib
    _lib.require_cuda()


def _policy(Do, Da, sizes, M, act='tanh', out=None, **kw):
    from promp_b200.policies import MetaGaussianMLPPolicy
    return MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=sizes,
                                 hidden_nonlinearity=act, output_nonlinearity=out, **kw)


class Case(object):
    """float32 inputs of one launch and the policy whose entry points run it (theta per task, or shared)."""

    def __init__(self, Do, Da, sizes, M, N, seed, act='tanh', out=None, shared=False, n_valid=None, explore=False):
        rng = np.random.RandomState(seed)
        self.Do, self.Da, self.sizes, self.M, self.N, self.act, self.out = Do, Da, tuple(sizes), M, N, act, out
        self.dims = (Do, Da, self.sizes)
        self.shared, self.n_valid, self.explore = shared, n_valid, explore
        PL = n_logical(*self.dims)
        self.ls_lo = PL - Da
        base = np.concatenate([rng.uniform(-1, 1, int(np.prod(s))) * math.sqrt(3.0 / (s[0] + s[-1])) if len(s) == 2 and 'kernel' in n
                               else 0.1 * rng.randn(int(np.prod(s))) for n, s in ref_shapes(*self.dims)])
        theta = np.repeat(base[None], M, 0) if shared else base[None] + 0.05 * rng.randn(M, PL)
        theta[:, self.ls_lo:] = rng.uniform(-0.7, 0.3, size=Da)
        self.theta_tasks = theta.astype(np.float32)
        obs = rng.randn(M, N, Do)
        with torch.no_grad():
            mean, _ = dist_info(torch.from_numpy(self.theta_tasks).double(), torch.from_numpy(obs.astype(np.float32)).double(),
                                self.dims, act, out)
        old_mean = mean.numpy() + 0.2 * rng.randn(M, N, Da)
        old_ls = self.theta_tasks[:, self.ls_lo:] + 0.1 * rng.randn(M, Da)
        act_ = old_mean + np.exp(old_ls)[:, None] * rng.randn(M, N, Da)
        f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)      # noqa: E731
        self.obs, self.act_s, self.old_mean, self.old_ls = f32(obs), f32(act_), f32(old_mean), f32(old_ls)
        self.adv = f32(rng.randn(M)) if explore else f32(rng.randn(M, N))
        self.vec_np = f32(0.3 * rng.randn(M, PL))
        self.pol = _policy(Do, Da, self.sizes, M, act, out)
        assert self.pol.num_params_logical == PL

    def data(self, m, n):
        t = lambda a: torch.from_numpy(np.array(a)).double()      # noqa: E731
        adv = np.full((1, n), self.adv[m]) if self.explore else self.adv[m:m + 1, :n]
        return dict(obs=t(self.obs[m:m + 1, :n]), act=t(self.act_s[m:m + 1, :n]), adv=t(adv), mean=t(self.old_mean[m:m + 1, :n]),
                    log_std=t(np.broadcast_to(self.old_ls[m:m + 1, None], (1, n, self.Da))))

    def per_task(self, fn):
        outs = []
        for m in range(self.M):
            n = self.N if self.n_valid is None else self.n_valid[m]
            outs.append(fn(torch.from_numpy(self.theta_tasks[m:m + 1]).double(), self.data(m, n), m))
        return [torch.cat(x, 0).numpy() for x in zip(*outs)]

    # ---- device
    def launch(self, kind, clip=1, kl_coeff=0.0, inner_lr=0.1, step_size=None):
        from promp_b200 import _lib
        pol, M, P = self.pol, self.M, self.pol.num_params
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
        params = dev(pol.pad_flat(self.theta_tasks[0] if self.shared else self.theta_tasks))
        obs, act, adv, mean = self.obs.copy(), self.act_s.copy(), self.adv.copy(), self.old_mean.copy()
        if self.n_valid is not None:       # poison in the padding rows
            for m, n in enumerate(self.n_valid):
                obs[m, n:] = 1e3; act[m, n:] = -50.0; mean[m, n:] = 7.0
                if not self.explore:
                    adv[m, n:] = 1e4
        bufs = [dev(a) for a in (obs, act, adv, mean, self.old_ls)]
        n_valid = None if self.n_valid is None else torch.tensor(self.n_valid, dtype=torch.int32, device='cuda')
        need = getattr(_lib.load(), pol.entries['workspace_bytes'])(M, self.N, self.Do, self.Da, pol.hidden_arg)
        ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device='cuda')
        p = _lib.ptr
        stats = torch.full((M, 4), float('nan'), device='cuda')
        stride = 0 if self.shared else P
        if kind == 'hvp':
            v = dev(pol.pad_flat(self.vec_np))
            out = torch.full((M, P), float('nan'), device='cuda')
            _lib.call(pol.entries['hvp_ragged'], self.Do, self.Da, pol.hidden_arg, M, self.N, p(n_valid), p(params), stride,
                      *[p(b) for b in bufs], 0, OBJ['ratio'], float(inner_lr), float(kl_coeff), int(clip), MIN_LOG_STD,
                      p(v), p(out), p(stats), p(ws), ws.numel() * 4, _lib.stream())
            torch.cuda.synchronize()
            return v, out, stats
        grad = torch.full((M, P), float('nan'), device='cuda')
        newp = torch.full((M, P), float('nan'), device='cuda')
        _lib.call(pol.entries['grad_ex'], self.Do, self.Da, pol.hidden_arg, M, self.N, p(n_valid), p(params), stride,
                  *[p(b) for b in bufs], 0, OBJ[kind], 1.0, CLIP_EPS, float(kl_coeff), int(clip), MIN_LOG_STD, p(grad),
                  p(newp) if kind != 'explore' else None, 0.1, p(stats), None, None, None, None, p(ws), ws.numel() * 4,
                  _lib.stream())
        torch.cuda.synchronize()
        return grad, newp, stats

    def pads(self, t):
        mask = np.ones(self.pol.num_params, dtype=bool)
        mask[self.pol._pad_index_np] = False
        return t.cpu().numpy()[:, mask]


def check_grad(c, kind, kl_coeff=0.2):
    grad, newp, stats = c.launch(kind, kl_coeff=kl_coeff)
    okind = 'loglik' if kind == 'explore' else kind
    want, st = c.per_task(lambda t, d, m: oracle_grad(t, d, c.dims, okind, c.act, c.out, kl_coeff, MIN_LOG_STD))
    assert np.all(c.pads(grad) == 0.0), 'pad entries of the gradient'
    assert_blocks('%s gradient' % kind, c.pol.unpad_flat(grad.cpu().numpy()), want, c.dims)
    np.testing.assert_allclose(stats.cpu().numpy()[:, :3], st, rtol=1e-4, atol=1e-6)
    if kind != 'explore':
        prm = c.pol.pad_flat(c.theta_tasks)
        prm = np.broadcast_to(prm[:1], prm.shape) if c.shared else prm
        np.testing.assert_allclose(newp.cpu().numpy(), prm - np.float32(0.1) * grad.cpu().numpy(), rtol=1e-6, atol=1e-7)


def check_hvp(c, kl_coeff=5e-4, inner_lr=0.1):
    v, out, stats = c.launch('hvp', kl_coeff=kl_coeff, inner_lr=inner_lr)
    want, = c.per_task(lambda t, d, m: (oracle_hvp_delta(t, d, c.dims, 'ratio', c.act, c.out,
                                                         torch.from_numpy(c.vec_np[m:m + 1]).double(), inner_lr, kl_coeff,
                                                         MIN_LOG_STD),))
    assert np.all(c.pads(out) == c.pads(v)), 'out != vec on pad entries'
    delta = c.pol.unpad_flat(out.cpu().numpy()).astype(np.float64) - c.vec_np.astype(np.float64)
    assert_blocks('HVP (out - vec)', delta, want, c.dims)


SHAPES = [(2, 2), (17, 6), (5, 3), (19, 8)]         # exact and bucket
DEEP_SIZES = {(1, 64): (64,), (1, 32): (32,), (3, 64): (64, 64, 64), (3, 32): (32, 32, 32)}


@pytest.mark.gpu
@pytest.mark.parametrize('out', [None, 'tanh'])
@pytest.mark.parametrize('act', ['tanh', 'relu'])
@pytest.mark.parametrize('hidden', [64, 32])
@pytest.mark.parametrize('depth', [1, 3])
@pytest.mark.parametrize('Do,Da', SHAPES)
def test_gradient_and_hvp_match_float64(Do, Da, depth, hidden, act, out):
    """Per task and block: ratio, log-likelihood and clipped gradients with the KL term, and the HVP, per-task parameters."""
    _cuda()
    c = Case(Do, Da, DEEP_SIZES[depth, hidden], 5, 200, seed=Do * 100 + Da * 10 + depth + hidden, act=act, out=out)
    assert c.pol.entries['grad_ex'].endswith('_padded') == ((Do, Da) not in EXACT_SHAPES)
    for kind in ('ratio', 'loglik', 'clip'):
        check_grad(c, kind)
    check_hvp(c)


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 63, 65, 257])
@pytest.mark.parametrize('depth', [1, 3])
def test_tile_edges_ragged_shared_and_explore(depth, N):
    """Partial tiles, variable-length paths (poison in the padding rows), shared parameters, the E-MAML exploration
    objective, and uneven widths padded to the widest layer."""
    _cuda()
    sizes = (64,) if depth == 1 else (64, 32, 16)
    c = Case(17, 6, sizes, 3, N, seed=N + depth)
    check_grad(c, 'ratio')
    check_hvp(c)
    if N > 1:
        cr = Case(5, 3, sizes, 4, N, seed=7 * N + depth, n_valid=[N, max(1, N // 2), 1, N - 1], act='relu')
        check_grad(cr, 'loglik')
        check_hvp(cr)
    cs = Case(2, 2, sizes, 3, N, seed=3 * N + depth, shared=True, explore=True)
    check_grad(cs, 'explore', kl_coeff=0.0)


@pytest.mark.gpu
def test_meta_sgd_step_sizes_in_the_deep_kernels():
    """Per-parameter inner step sizes (Meta-SGD): out_params = params - alpha * grad; the HVP is applied to alpha * vec."""
    _cuda()
    from promp_b200 import _lib
    c = Case(17, 6, (32, 32, 32), 3, 130, seed=5)
    pol, M, P = c.pol, c.M, c.pol.num_params
    alpha = torch.from_numpy(pol.pad_flat(np.random.RandomState(1).uniform(0.05, 0.2, pol.num_params_logical))).cuda()
    stage_g, stage_h = _lib.PolicyStage(), _lib.PolicyStage()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
    params, obs, act, adv, mean, ls = (dev(pol.pad_flat(c.theta_tasks)), dev(c.obs), dev(c.act_s), dev(c.adv), dev(c.old_mean),
                                       dev(c.old_ls))
    grad, newp = torch.zeros(M, P, device='cuda'), torch.zeros(M, P, device='cuda')
    vec, out = dev(pol.pad_flat(c.vec_np)), torch.zeros(M, P, device='cuda')
    p = _lib.ptr
    for st, kind in ((stage_g, 0), (stage_h, 1)):
        st.kind, st.N, st.params, st.param_stride = kind, c.N, p(params), P
        st.obs, st.act, st.adv, st.old_mean, st.old_log_std = p(obs), p(act), p(adv), p(mean), p(ls)
        st.obj_kind, st.obj_scale, st.clip_log_std, st.step_size = 0, 1.0, 1, p(alpha)
    stage_g.grad, stage_g.out_params = p(grad), p(newp)
    stage_h.inner_lr, stage_h.vec, stage_h.out = 1.0, p(vec), p(out)
    import ctypes
    for st in (stage_g, stage_h):
        arr = (_lib.PolicyStage * 1)(st)
        need = getattr(_lib.load(), pol.entries['chain_workspace_bytes'])(c.Do, c.Da, pol.hidden_arg, M, 1, ctypes.cast(arr, ctypes.c_void_p))
        ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device='cuda')
        _lib.call(pol.entries['chain'], c.Do, c.Da, pol.hidden_arg, M, MIN_LOG_STD, 1, ctypes.cast(arr, ctypes.c_void_p), None,
                  None, p(ws), ws.numel() * 4, _lib.stream())
    torch.cuda.synchronize()
    np.testing.assert_allclose(newp.cpu().numpy(), pol.pad_flat(c.theta_tasks) - alpha.cpu().numpy() * grad.cpu().numpy(),
                               rtol=1e-6, atol=1e-7)
    a_l = pol.unpad_flat(alpha.cpu().numpy()).astype(np.float64)
    want, = c.per_task(lambda t, d, m: (oracle_hvp_delta(t, d, c.dims, 'ratio', c.act, c.out,
                                                         torch.from_numpy(a_l * c.vec_np[m:m + 1]).double(), 1.0, 0.0,
                                                         MIN_LOG_STD),))
    delta = pol.unpad_flat(out.cpu().numpy()).astype(np.float64) - c.vec_np.astype(np.float64)
    assert_blocks('Meta-SGD HVP', delta, want, c.dims)


# ------------------------------------------------------------------------------------------------ chain / meta-gradient
def _meta_grad_oracle(c, inner_steps, inner_lr, kl_coeff=0.0):
    """d/dtheta of the ProMP clipped outer objective at theta_S = theta - inner_lr * grad(inner ratio surr) applied S times
    (the same phase data every step), per task, float64."""
    outs = []
    for m in range(c.M):
        d = c.data(m, c.N)
        t = torch.from_numpy(c.theta_tasks[m:m + 1]).double().requires_grad_(True)
        x = t
        for _ in range(inner_steps):
            surr, _, _ = terms(x, d, c.dims, 'ratio', c.act, c.out)
            (g,) = torch.autograd.grad(surr.sum(), x, create_graph=True)
            x = x - inner_lr * g
        surr, kl, _ = terms(x, d, c.dims, 'clip', c.act, c.out)
        (g,) = torch.autograd.grad((surr + kl_coeff * kl).sum(), t)
        outs.append(g)
    return torch.cat(outs).numpy()


@pytest.mark.gpu
@pytest.mark.parametrize('inner_steps', [1, 2])
@pytest.mark.parametrize('depth', [1, 3])
def test_chain_meta_gradient(depth, inner_steps):
    """promp_policy_chain with 2 S + 1 stages (inner gradients, outer gradient, HVP stages): one launch per stage, equal bit
    for bit to the stages launched separately, and the meta-gradient matches float64 autograd through the inner steps."""
    _cuda()
    import ctypes
    from promp_b200 import _lib
    c = Case(17, 6, DEEP_SIZES[depth, 64], 6, 300, seed=40 + depth + inner_steps)
    pol, M, P, N = c.pol, c.M, c.pol.num_params, c.N
    lr = 0.05
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
    obs, act, adv, mean, ls = dev(c.obs), dev(c.act_s), dev(c.adv), dev(c.old_mean), dev(c.old_ls)
    theta = dev(pol.pad_flat(c.theta_tasks))
    p = _lib.ptr

    def build():
        thetas = [theta] + [torch.zeros(M, P, device='cuda') for _ in range(inner_steps)]
        grads = [torch.zeros(M, P, device='cuda') for _ in range(inner_steps + 1)]
        outs = [torch.zeros(M, P, device='cuda') for _ in range(inner_steps)]
        st = []
        for s in range(inner_steps + 1):
            g = _lib.PolicyStage(kind=0, N=N, params=p(thetas[s]), param_stride=P, obs=p(obs), act=p(act), adv=p(adv),
                                 old_mean=p(mean), old_log_std=p(ls), obj_kind=0 if s < inner_steps else 2, obj_scale=1.0,
                                 clip_eps=CLIP_EPS, clip_log_std=0, grad=p(grads[s]),
                                 out_params=p(thetas[s + 1]) if s < inner_steps else None, sgd_lr=lr)
            st.append(g)
        v = grads[-1]
        for k, s in enumerate(reversed(range(inner_steps))):
            st.append(_lib.PolicyStage(kind=1, N=N, params=p(thetas[s]), param_stride=P, obs=p(obs), act=p(act), adv=p(adv),
                                       old_mean=p(mean), old_log_std=p(ls), obj_kind=0, clip_log_std=0, inner_lr=lr,
                                       vec=p(v), out=p(outs[k])))
            v = outs[k]
        return st, v

    stages, result = build()
    arr = (_lib.PolicyStage * len(stages))(*stages)
    sp = ctypes.cast(arr, ctypes.c_void_p)
    n = len(stages)
    assert getattr(_lib.load(), pol.entries['chain_num_launches'])(c.Do, c.Da, pol.hidden_arg, M, n, sp) == n
    need = getattr(_lib.load(), pol.entries['chain_workspace_bytes'])(c.Do, c.Da, pol.hidden_arg, M, n, sp)
    ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device='cuda')
    _lib.call(pol.entries['chain'], c.Do, c.Da, pol.hidden_arg, M, MIN_LOG_STD, n, sp, None, None, p(ws), ws.numel() * 4,
              _lib.stream())
    torch.cuda.synchronize()
    chain_out = result.clone()
    # the same stages as stand-alone launches
    stages2, result2 = build()
    need1 = getattr(_lib.load(), pol.entries['workspace_bytes'])(M, N, c.Do, c.Da, pol.hidden_arg)
    ws1 = torch.zeros((need1 + 3) // 4, dtype=torch.int32, device='cuda')
    for g in stages2:
        if g.kind == 0:
            _lib.call(pol.entries['grad_ex'], c.Do, c.Da, pol.hidden_arg, M, N, None, g.params, P, g.obs, g.act, g.adv, g.old_mean,
                      g.old_log_std, 0, g.obj_kind, 1.0, CLIP_EPS, 0.0, 0, MIN_LOG_STD, g.grad, g.out_params, lr, None, None, None,
                      None, None, p(ws1), ws1.numel() * 4, _lib.stream())
        else:
            _lib.call(pol.entries['hvp_ragged'], c.Do, c.Da, pol.hidden_arg, M, N, None, g.params, P, g.obs, g.act, g.adv,
                      g.old_mean, g.old_log_std, 0, 0, lr, 0.0, 0, MIN_LOG_STD, g.vec, g.out, None, p(ws1), ws1.numel() * 4,
                      _lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(chain_out, result2)
    want = _meta_grad_oracle(c, inner_steps, lr)
    assert np.all(c.pads(chain_out) == 0.0)
    assert_blocks('meta-gradient (%d inner steps)' % inner_steps, pol.unpad_flat(chain_out.cpu().numpy()), want, c.dims)


# ------------------------------------------------------------------------------------------------ forward / get_actions
@pytest.mark.gpu
@pytest.mark.parametrize('sizes', [(64,), (32,), (64, 64, 64), (32, 16, 8)])
@pytest.mark.parametrize('Do,Da', [(17, 6), (5, 3), (2, 2)])
def test_get_actions_and_forward(Do, Da, sizes):
    _cuda()
    for act, out in (('tanh', None), ('relu', 'tanh')):
        pol = _policy(Do, Da, sizes, 3, act, out)
        obs = [np.random.RandomState(m).randn(70, Do).astype(np.float32) for m in range(3)]
        _, infos = pol.get_actions(obs)
        theta = torch.from_numpy(pol.unpad_flat(pol.theta.cpu().numpy())).double()[None].expand(3, -1)
        want, _ = dist_info(theta, torch.from_numpy(np.stack(obs)).double(), (Do, Da, sizes), act, out)
        got = np.stack([[infos[m][e]['mean'] for e in range(70)] for m in range(3)])
        np.testing.assert_allclose(got, want.numpy(), rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_policy_constructor_names_and_pickle():
    _cuda()
    from promp_b200 import _lib
    for bad in ((), (64, 64, 64, 64), (32,) * 5):
        with pytest.raises(NotImplementedError, match='1 to 3 hidden layers'):
            _policy(2, 2, bad, 2)
    for sizes in ((64,), (32, 32), (64, 32, 16)):
        pol = _policy(17, 6, sizes, 2, 'relu')
        assert list(pol.param_shapes.items()) == ref_shapes(17, 6, sizes)
        assert pol.policy_params_keys == [n for n, _ in ref_shapes(17, 6, sizes)]
        assert pol.hidden_arg == (32 if max(sizes) <= 32 else 64) | _lib.ACT_RELU | _lib.hidden_depth(len(sizes))
        pol2 = pickle.loads(pickle.dumps(pol))
        assert pol2.hidden_arg == pol.hidden_arg and torch.equal(pol2.theta, pol.theta)
        assert list(pol2.get_param_values()) == list(pol.get_param_values())
    assert _policy(2, 2, (32, 32), 2).hidden_arg == 32


# ------------------------------------------------------------------------------------------------ fused rollout
ROLLOUT_ENVS = dict(point_corner=(0, 2, 2, 2, False), point=(1, 2, 2, 1, True), cheetah=(2, 17, 6, 1, False),
                    swimmer=(6, 8, 2, 1, False), walker=(5, 17, 6, 2, True))


def _rollout(kind, early, M, E, T, H, hidden_arg, params, PL, task_d, noise_d, bufs, task_offset=0):
    from promp_b200 import _lib
    obs, act, mean, rew, done, info, ls_out = bufs
    p = _lib.ptr
    if early:
        _lib.call('promp_rollout_early_term_ex', kind, 1, M, E, T, H, hidden_arg, p(params), PL, p(task_d), None, p(noise_d),
                  5, 1, None, 0, -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(ls_out), _lib.stream(), task_offset)
    else:
        _lib.call('promp_rollout_ex', kind, 0 if kind != 0 else 1, 0.5, 1, M, E, H, hidden_arg, p(params), PL, p(task_d), None,
                  p(noise_d), 5, 1, None, 0, -13.8, p(obs), p(act), p(mean), p(rew), p(done), p(info), p(ls_out), None,
                  _lib.stream(), task_offset)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('act,out', [('tanh', None), ('relu', 'tanh')])
@pytest.mark.parametrize('hidden', [64, 32])
@pytest.mark.parametrize('depth', [1, 3])
@pytest.mark.parametrize('env', list(ROLLOUT_ENVS))
def test_fused_rollout_teacher_forced(env, depth, hidden, act, out):
    """promp_rollout_ex / promp_rollout_early_term_ex (plain and sharded) with fed noise: the recorded means against the
    float64 policy on the kernel's own observations, act = mean + eps * exp(log_std)."""
    _cuda()
    from promp_b200 import _lib
    kind, Do, Da, TD, early = ROLLOUT_ENVS[env]
    M, E, H = 3, 6, 40
    rng = np.random.RandomState(kind * 10 + hidden + depth)
    sizes = (hidden,) * depth
    pol = _policy(Do, Da, sizes, M, act, out)
    PL = pol.num_params
    theta_l = np.stack([pol.unpad_flat(pol.theta.cpu().numpy())] * M).astype(np.float64)
    theta_l += 0.1 * rng.randn(*theta_l.shape)
    theta_l[:, -Da:] = -0.5
    theta_l = theta_l.astype(np.float32)
    if kind == 2:
        task = rng.choice([-1.0, 1.0], size=(M, 1))
    elif kind == 5:
        task = np.stack([rng.uniform(0, 2, M), rng.randint(0, 2, M)], 1)
    else:
        task = rng.uniform(-1, 1, size=(M, TD))
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()       # noqa: E731
    T = 2 * H - 1 if early else H
    noise = rng.randn(M, E, T, Da).astype(np.float32)
    bufs = tuple(torch.empty(M, E, T, n, device='cuda') for n in (Do, Da, Da)) + (
        torch.empty(M, E, T, device='cuda'), torch.empty(M, E, T, dtype=torch.uint8, device='cuda'),
        torch.zeros(3, M, E, T, device='cuda'), torch.empty(M, Da, device='cuda'))
    params, task_d, noise_d = dev(pol.pad_flat(theta_l)), dev(task), dev(noise)
    for task_offset in (0, 2):
        _rollout(kind, early, M, E, T, H, pol.hidden_arg, params, PL, task_d, noise_d, bufs, task_offset)
        o, a, mu = (b.cpu().numpy() for b in bufs[:3])
        if early:
            assert bufs[4].cpu().numpy().sum() >= M * E
        want, _ = dist_info(torch.from_numpy(theta_l).double(), torch.from_numpy(o.reshape(M, E * T, Do)).double(),
                            (Do, Da, sizes), act, out)
        np.testing.assert_allclose(mu, want.numpy().reshape(M, E, T, Da), rtol=1e-4, atol=2e-5)
        sig = np.exp(theta_l[:, -Da:].astype(np.float64))[:, None, None, :]
        np.testing.assert_allclose(a, mu + noise * sig, rtol=1e-5, atol=1e-5)
        np.testing.assert_array_equal(bufs[6].cpu().numpy(), theta_l[:, -Da:])


@pytest.mark.gpu
@pytest.mark.parametrize('keyed', [0, 2])
def test_user_env_rollout_with_a_deep_policy(tmp_path, monkeypatch, keyed):
    """A CudaMetaEnv (the cheetah through the warp concept, compiled by NVRTC) with a three-layer policy: its module's
    rollout_deep_kernel records what the library's built-in kernel records (bit for bit when NVRTC is the library's CUDA
    version), plain and sharded."""
    _cuda()
    monkeypatch.setenv('PROMP_B200_JIT_CACHE', str(tmp_path / 'jit'))
    from promp_b200 import _jit, _lib
    from promp_b200.envs import CudaMetaEnv, HalfCheetahRandDirecEnv, normalize
    inner = HalfCheetahRandDirecEnv()
    twin = CudaMetaEnv('', obs_dim=inner.obs_dim, act_dim=inner.act_dim, state_dim=18, task_dim=1,
                       action_space=inner.action_space, sample_tasks=inner.sample_tasks, task_vector=inner.task_vector,
                       host_reset_states=inner.host_reset_states, info_keys=('reward_run', 'reward_ctrl'),
                       struct_name='promp::Cheetah')
    M, E, H = 4, 8, 50
    pol = _policy(17, 6, (64, 64, 64), M)
    module = normalize(twin).device_spec()['module'].handle(pol.hidden_arg)
    rng = np.random.RandomState(2)
    task = torch.from_numpy(rng.choice([-1.0, 1.0], size=(M, 1)).astype(np.float32)).cuda()
    p = _lib.ptr
    outs = []
    for entry, first in (('promp_rollout_ex', _lib.ENV_CHEETAH_DIR), ('promp_rollout_module', module)):
        f = lambda *sh: torch.full(sh, float('nan'), device='cuda')     # noqa: E731
        o = dict(obs=f(M, E, H, 17), act=f(M, E, H, 6), mean=f(M, E, H, 6), rew=f(M, E, H), info=f(3, M, E, H), ls=f(M, 6),
                 fs=f(M, E, 18), done=torch.zeros(M, E, H, dtype=torch.uint8, device='cuda'))
        _lib.call(entry, first, 0, 0.5, 1, M, E, H, pol.hidden_arg, p(pol.theta), 0, p(task), None, None, 9, 3, None, 1,
                  float(pol.min_log_std), p(o['obs']), p(o['act']), p(o['mean']), p(o['rew']), p(o['done']), p(o['info']),
                  p(o['ls']), p(o['fs']), _lib.stream(), keyed)
        torch.cuda.synchronize()
        outs.append({k: v.cpu().numpy() for k, v in o.items()})
    for k in ('obs', 'act', 'mean', 'rew', 'done', 'ls', 'fs'):
        a, b = outs[1][k], outs[0][k]
        assert np.all(np.isfinite(a.astype(np.float64))), k
        if _jit.matches_library():
            assert np.array_equal(a, b), k
        else:
            np.testing.assert_allclose(a, b, rtol=1e-4, atol=1e-4, err_msg=k)


# ------------------------------------------------------------------------------------------------ Trainer
def _trainer(algo_kind, env_kind, depth, graph, seed=11, M=4, E=3, H=30):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnvCorner, HalfCheetahRandDirecEnv
    from promp_b200.meta_algos import ProMP, TRPOMAML, VPGMAML
    from promp_b200.meta_trainer import Trainer
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    np.random.seed(seed)
    torch.manual_seed(seed)
    env = normalize(MetaPointEnvCorner(reward_type='dense') if env_kind == 'point' else HalfCheetahRandDirecEnv())
    Do, Da = int(np.prod(env.observation_space.shape)), int(np.prod(env.action_space.shape))
    policy = _policy(Do, Da, (64,) if depth == 1 else (64, 32, 32), M)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    if algo_kind == 'promp':
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=3, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    elif algo_kind == 'trpo':
        algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, step_size=0.01)
    else:
        algo = VPGMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3)
    return Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                   num_inner_grad_steps=1, use_cuda_graph=graph)


def _train(tr, tmp_path):
    from promp_b200.utils import logger
    policy = tr.policy
    theta0 = policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='last')
        tr.train()
        kv = dict(logger.last_dump())
    finally:
        logger.reset()
    assert not torch.equal(policy.theta, theta0) and torch.isfinite(policy.theta).all()
    mask = np.ones(policy.num_params, dtype=bool)
    mask[policy._pad_index_np] = False
    assert np.all(policy.theta.cpu().numpy()[mask] == 0.0), 'pad entries left zero'
    return kv


@pytest.mark.gpu
@pytest.mark.parametrize('algo', ['promp', 'trpo', 'vpg'])
@pytest.mark.parametrize('env', ['point', 'cheetah'])
@pytest.mark.parametrize('depth', [1, 3])
def test_trainer_runs(depth, env, algo, tmp_path):
    """Three meta-iterations of Trainer.train() in CUDA-graph mode (ProMP, TRPO-MAML; VPG-MAML has no device-only outer step
    and runs eagerly) and eagerly: every logged scalar finite, pad entries (the uneven widths of (64, 32, 32)) exactly zero
    through the Adam / TRPO steps, and the same seed gives the same run bit for bit."""
    _cuda()
    runs = []
    for i, graph in enumerate((True, True, False)):
        tr = _trainer(algo, env, depth, graph and algo != 'vpg')
        if graph and algo != 'vpg':
            assert tr.graph_capturable()
        runs.append((tr.policy.theta.clone(), _train(tr, tmp_path / str(i))))
    kv = runs[0][1]
    assert kv['Itr'] == 2
    assert all(np.isfinite(v) for k, v in kv.items() if isinstance(v, (float, int, np.floating)) and 'Time' not in k)
    assert torch.equal(runs[0][0], runs[1][0])
    for k, v in kv.items():
        if 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert v == runs[1][1][k], k


@pytest.mark.gpu
@pytest.mark.parametrize('algo', ['promp', 'trpo'])
@pytest.mark.parametrize('depth', [1, 3])
def test_graph_replayed_step_equals_eager(depth, algo):
    """The device part of a meta-iteration (optimize_phases) of a deep policy captured as a CUDA graph and replayed gives
    the parameters and logged terms of the eager call on the same phases, bit for bit.  (The Trainer's eager and graph
    modes draw their action noise from differently keyed streams, so whole runs are compared per mode above.)"""
    _cuda()
    tr = _trainer(algo, 'cheetah', depth, False)
    sampler, proc, algo_, policy = tr.sampler, tr.sample_processor, tr.algo, tr.policy
    sampler.update_tasks()
    policy.switch_to_pre_update()
    samples = []
    for step in range(2):
        s = proc.process_samples(sampler.obtain_samples())
        samples.append(s)
        if step == 0:
            algo_._adapt(s)
    phases = [s[0].phase for s in samples]
    theta0 = policy.theta.clone()
    opt_slots = getattr(algo_.optimizer, 'slots', lambda: [])()     # ProMP's Adam state: every call starts from the same one
    slots0 = [t.clone() for t in opt_slots]

    def reset():
        policy.theta.copy_(theta0)
        for t, t0 in zip(opt_slots, slots0):
            t.copy_(t0)
    algo_._adapt_cache = None
    eager = algo_.optimize_phases(phases).clone()
    th_eager = policy.theta.clone()
    for ph in phases:
        ph.invalidate_host()
    reset()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        algo_.optimize_phases(phases)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for ph in phases:
        ph.invalidate_host()
    reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = algo_.optimize_phases(phases)
    reset()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager), (out, eager)
    assert torch.equal(policy.theta, th_eager)
    assert not torch.equal(th_eager, theta0)


# ------------------------------------------------------------------------------------------------ reference graph (golden)
# tests/golden/tf_half_depth.npz: the reference's unmodified TF1 graph code for one and three hidden layers, evaluated in
# float64 on the torch-backed stand-in of oracle/stubs_tf (tools/make_depth_golden.py; the cases' inputs are stored with it)
GOLDEN = ('promp_d1_h64', 'promp_d1_h32', 'promp_d3_h64', 'promp_d3_uneven', 'trpo_d1_h64', 'trpo_d3_uneven')
GOLDEN_DIMS = dict(promp_d1_h64=(2, 2, (64,)), promp_d1_h32=(17, 6, (32,)), promp_d3_h64=(2, 2, (64, 64, 64)),
                   promp_d3_uneven=(5, 3, (32, 16, 8)), trpo_d1_h64=(2, 2, (64,)), trpo_d3_uneven=(5, 3, (32, 16, 8)))
INNER_LR = float(np.float32(0.1))       # the reference's inner_lr is a float32 constant


@pytest.fixture(scope='module')
def depth_gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'tf_half_depth.npz'))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _gold_phases(G, name, dt=torch.float64):
    out = []
    for s in range(2):
        g = lambda k: torch.tensor(G['%s/phase%d_%s' % (name, s, k)], dtype=dt)      # noqa: E731
        N = G['%s/phase%d_obs' % (name, s)].shape[1]
        out.append(dict(obs=g('obs'), act=g('act'), adv=g('adv'), mean=g('mean'), log_std=g('log_std')[:, None, :].expand(-1, N, -1),
                        adj_avg_rewards=torch.zeros_like(g('adv'))))
    return out


@contextlib.contextmanager
def _depth_oracle(monkeypatch):
    """oracle/tf_half's ProMP / TRPO-MAML objective with the depth-generic policy forward."""
    def di(theta, obs, dims, min_log_std=None):
        mean, ls = dist_info(theta, obs, dims)
        return mean, (torch.clamp(ls, min=min_log_std) if min_log_std is not None else ls)
    monkeypatch.setattr(th, 'dist_info', di)
    yield


@pytest.mark.parametrize('name', GOLDEN)
def test_float64_oracle_reproduces_reference_graph(depth_gold, name, monkeypatch):
    """The float64 depth-generic policy inside oracle/tf_half's meta objective == the reference graph: the adapt step, the
    second-order ProMP meta-gradient, its loss and KLs and one TF1 Adam step, and TRPO-MAML's objective and KL gradients."""
    G, dims = depth_gold, GOLDEN_DIMS[name]
    with _depth_oracle(monkeypatch):
        data = _gold_phases(G, name)
        theta = torch.tensor(G[name + '/theta'], dtype=torch.float64)
        M = data[0]['obs'].shape[0]
        cur = th.adapt(theta[None].expand(M, -1).contiguous(), data[0], dims, INNER_LR)
        assert _rel(cur.numpy() - G[name + '/theta'].astype(np.float64), G[name + '/adapt_delta']) < 1e-6
        algo = 'promp' if name.startswith('promp') else 'trpo'
        t = theta.clone().requires_grad_(True)
        obj, ikl, okl = th.meta_objective(t, data, dims, INNER_LR, algo, 0.3, [5e-4])
        (g,) = torch.autograd.grad(obj, t)
        assert abs(float(obj.detach()) - float(G[name + '/loss'])) <= 1e-9 + 1e-6 * abs(float(G[name + '/loss']))
        assert _rel(g.numpy(), G[name + '/grad']) < 1e-6
        assert abs(float(okl.detach()) - float(G[name + '/outer_kl'])) <= 1e-12 + 1e-5 * abs(float(G[name + '/outer_kl']))
        if algo == 'promp':
            np.testing.assert_allclose(ikl.detach().numpy(), G[name + '/inner_kl'], rtol=1e-5, atol=1e-12)
            adam = th.TF1Adam(theta.numel(), lr=1e-3, dtype=torch.float64)
            new = adam.step(theta, g)
            assert _rel(new.numpy() - theta.numpy(), G[name + '/adam_theta'].astype(np.float64) - G[name + '/theta']) < 1e-4
        else:
            t = theta.clone().requires_grad_(True)
            (gk,) = torch.autograd.grad(th.meta_objective(t, data, dims, INNER_LR, 'trpo')[2], t)
            assert _rel(gk.numpy(), G[name + '/kl_grad']) < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize('name', GOLDEN)
def test_product_matches_reference_graph(depth_gold, name):
    """MAMLAlgo._adapt, the meta-gradient (ProMP through the chain entry point, TRPO-MAML through its gradient passes) and
    one device Adam step (promp_adam_tf1) against the reference graph, within 1e-4 relative."""
    _cuda()
    from collections import OrderedDict
    from promp_b200 import _lib
    from promp_b200.meta_algos import ProMP, TRPOMAML
    G, (Do, Da, sizes) = depth_gold, GOLDEN_DIMS[name]
    theta0 = G[name + '/theta'].astype(np.float64)
    M = G[name + '/phase0_obs'].shape[0]
    np.random.seed(1)
    policy = _policy(Do, Da, sizes, M)
    flat, off = OrderedDict(), 0
    for k, shp in ref_shapes(Do, Da, sizes):
        n = int(np.prod(shp))
        flat[k] = G[name + '/theta'][off:off + n].reshape(shp)
        off += n
    policy.set_params(flat)
    if name.startswith('promp'):
        algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                     num_ppo_steps=1, clip_eps=0.3, target_inner_step=0.01, init_inner_kl_penalty=5e-4,
                     adaptive_inner_kl_penalty=False)
    else:
        algo = TRPOMAML(policy=policy, step_size=0.01, inner_type='likelihood_ratio', inner_lr=0.1, meta_batch_size=M,
                        num_inner_grad_steps=1)
    samples = []
    for s in range(2):
        g = lambda k: G['%s/phase%d_%s' % (name, s, k)]      # noqa: E731
        N = g('obs').shape[1]
        samples.append([dict(observations=g('obs')[m], actions=g('act')[m], advantages=g('adv')[m],
                             adj_avg_rewards=np.zeros(N, np.float32),
                             agent_infos=dict(mean=g('mean')[m], log_std=np.tile(g('log_std')[m][None], (N, 1))))
                        for m in range(M)])
    policy.switch_to_pre_update()
    algo._adapt(samples[0])
    delta = policy.unpad_flat(policy.theta_tasks.cpu().numpy()).astype(np.float64) - theta0[None]
    assert _rel(delta, G[name + '/adapt_delta']) < 1e-4
    phases = [algo._phase_of(s) for s in samples]
    if name.startswith('trpo'):
        g_got = policy.unpad_flat(np.asarray(algo.eval_gradient(policy.theta, phases, 'loss'), np.float64))
        gk = policy.unpad_flat(np.asarray(algo.eval_gradient(policy.theta, phases, 'kl'), np.float64))
        assert _rel(gk, G[name + '/kl_grad']) < 1e-4
        assert _rel(g_got, G[name + '/grad']) < 1e-4
        return
    res = algo._objective_pass(phases, want_grad=True)
    grad = res['grad']
    loss = float(algo.loss_terms(res).cpu().numpy()[0])
    assert abs(loss - float(G[name + '/loss'])) <= 2e-6 + 1e-4 * abs(float(G[name + '/loss']))
    assert _rel(policy.unpad_flat(grad.cpu().numpy()), G[name + '/grad']) < 1e-4
    P = policy.num_params
    theta = policy.theta.clone()
    m_, v_ = torch.zeros(P, device='cuda'), torch.zeros(P, device='cuda')
    step = torch.zeros(1, dtype=torch.int32, device='cuda')
    p = _lib.ptr
    _lib.call('promp_adam_tf1', P, p(theta), p(grad.contiguous()), p(m_), p(v_), p(step), 1e-3, 0.9, 0.999, 1e-8, _lib.stream())
    torch.cuda.synchronize()
    mask = np.ones(P, dtype=bool)
    mask[policy._pad_index_np] = False
    assert np.all(theta.cpu().numpy()[mask] == 0.0)
    got = policy.unpad_flat(theta.cpu().numpy()).astype(np.float64) - theta0
    assert _rel(got, G[name + '/adam_theta'].astype(np.float64) - theta0) < 1e-4
