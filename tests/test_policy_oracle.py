"""Policy gradient, Hessian-vector product and forward kernels against a float64 autograd oracle, per task and per
parameter block, at the tile and scheduling edges of the kernels.

The oracle is composed of the pinned functions of oracle/tf_half.py (dist_info, likelihood_ratio, log_likelihood, kl) and is
evaluated in float64 on the same float32 inputs the kernels get:
  gradient   d/dtheta of  obj_scale * surr_kind + kl_coeff * mean_n KL(old || new)   (surr_kind RATIO | LOGLIK | CLIP | NONE)
  stats      surr (unscaled), mean KL, mean ratio
  HVP        out - vec = -inner_lr * H vec + kl_coeff * grad mean KL, H = Hessian of the inner surrogate (double backward)
with max(log_std, min_log_std) when clip_log_std = 1 and a per-sample old log_std when ls_per_sample = 1.

Every result is split into the seven parameter blocks W0 b0 W1 b1 W2 b2 log_std (logical entries of the padded layouts)
and checked per task m and block b:
    |got - want|_mb <= RTOL |want_mb| + FLOOR |want_m|
W1 holds most of the parameters, so one norm over the whole vector would hide an error confined to a small block or to one
task.  Exact checks ride along: pad entries of every gradient are 0.0 and out == vec on them, clipped log_std components
get gradient 0.0 and out == vec, and out_params == params - sgd_lr * grad to one ulp of the kernel's own gradient.

CPU tests show that the bar is sound: the HVP oracle agrees with central differences of the oracle gradient, the same
oracle run in float32 passes the bar with a 10x margin (this sets FLOOR from below), and the bar rejects a set of small,
plausible kernel errors (this bounds FLOOR from above).  GPU tests (-m gpu) run the kernels.
"""
import contextlib
import math
import re

import numpy as np
import pytest
import torch

from oracle import tf_half as th

RTOL = 1e-4           # the project's parity bar
# Per-task floor for blocks whose value is small by cancellation (the KL-only gradient of log_std near the old policy is the
# worst).  Measured with test_float32_oracle_passes_with_margin: at FLOOR = 0 the float32 oracle's worst block error is 1.10x
# the bound (4x2 h64, KL-only gradient, log_std); at 2e-5 it is 0.071x (1x1 h64, HVP, W1): a 14x margin.  From above, the
# test_bar_rejects_* perturbations stay rejected up to a floor of 3.4e-5 (log_std of one task x (1 + 3e-4)).
FLOOR = 2e-5
BLOCKS = ('W0', 'b0', 'W1', 'b1', 'W2', 'b2', 'log_std')
OBJ = dict(ratio=0, loglik=1, clip=2, none=3)
CLIP_EPS = 0.3
DEFAULT_MIN_LOG_STD = math.log(1e-6)
EXACT_SHAPES = ((2, 2), (4, 2), (17, 6))
BUCKET_SHAPES = ((1, 1), (5, 3), (19, 8))
TILE_EDGE_N = (1, 63, 64, 65, 127, 128, 129, 256, 257)


# ------------------------------------------------------------------------------------------------------------ oracle
def _dims(Do, Da, hidden):
    return (Do, Da, (hidden, hidden))


def _block_slices(Do, Da, hidden):
    out, off = [], 0
    for shape in th.param_shapes(*_dims(Do, Da, hidden)).values():
        n = int(np.prod(shape))
        out.append(slice(off, off + n))
        off += n
    return out


def _terms(theta, d, dims, kind, clip_eps, min_log_std, straight_through_clip=False):
    """Per-task (surr, mean KL, mean ratio, mean |surr term|) at theta [M,P]; d holds obs / act / adv / mean / log_std [M,N,.]."""
    mean, ls = th.dist_info(theta, d['obs'], dims)
    if min_log_std is not None:
        clipped = torch.clamp(ls, min=min_log_std)
        # straight_through_clip: the clipped value forward, the unclipped gradient backward (a kernel that forgot the mask)
        ls = ls + (clipped - ls).detach() if straight_through_clip else clipped
    ratio = th.likelihood_ratio(d['act'], d['mean'], d['log_std'], mean, ls)
    adv = d['adv']
    if kind == 'ratio':
        per = ratio * adv
    elif kind == 'loglik':
        per = th.log_likelihood(d['act'], mean, ls) * adv
    elif kind == 'clip':
        per = torch.minimum(ratio * adv, torch.clamp(ratio, 1 - clip_eps, 1 + clip_eps) * adv)
    else:
        per = torch.zeros_like(adv)
    kl = torch.mean(th.kl(d['mean'], d['log_std'], mean, ls), -1)
    return -torch.mean(per, -1), kl, torch.mean(ratio, -1), torch.mean(per.abs(), -1)


def oracle_grad(theta, d, dims, kind, obj_scale=1.0, clip_eps=CLIP_EPS, kl_coeff=0.0, min_log_std=None, **kw):
    """(grad [M,P], stats [M,3] = surr, mean KL, mean ratio, stats scale [M,3]) in the dtype of theta."""
    t = theta.detach().clone().requires_grad_(True)
    surr, kl, ratio, surr_abs = _terms(t, d, dims, kind, clip_eps, min_log_std, **kw)
    (g,) = torch.autograd.grad((obj_scale * surr + kl_coeff * kl).sum(), t)
    stats = torch.stack([surr, kl, ratio], -1).detach()
    scale = torch.stack([surr_abs, kl.abs(), ratio.abs()], -1).detach()
    return g, stats, scale


def oracle_hvp_delta(theta, d, dims, kind, vec, inner_lr, kl_coeff, min_log_std=None, **kw):
    """out - vec = -inner_lr * H vec + kl_coeff * grad mean KL, per task [M,P]."""
    t = theta.detach().clone().requires_grad_(True)
    surr, kl, _, _ = _terms(t, d, dims, kind, 0.0, min_log_std, **kw)
    (g,) = torch.autograd.grad(surr.sum(), t, create_graph=True)
    (hv,) = torch.autograd.grad((g * vec).sum(), t, retain_graph=True)
    (gk,) = torch.autograd.grad(kl.sum(), t)
    return -inner_lr * hv + kl_coeff * gk


def oracle_ragged(fn, theta, d, n_valid, *args, **kw):
    """fn per task on its first n_valid[m] samples (the padding rows hold poison on the device only)."""
    outs = []
    for m, n in enumerate(n_valid):
        dm = {k: v[m:m + 1, :n] for k, v in d.items()}
        r = fn(theta[m:m + 1], dm, *args, **kw)
        outs.append(r if isinstance(r, tuple) else (r,))
    cat = tuple(torch.cat(x, 0) for x in zip(*outs))
    return cat if len(cat) > 1 else cat[0]


# -------------------------------------------------------------------------------------------------------- comparison
def block_ratios(got, want, Do, Da, hidden):
    """[M, 7]: |got - want|_mb / (RTOL |want_mb| + FLOOR |want_m|)  (<= 1 passes); got / want [M, P_logical]."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    norm_m = np.linalg.norm(want, axis=1)
    out = np.zeros((want.shape[0], len(BLOCKS)))
    for b, sl in enumerate(_block_slices(Do, Da, hidden)):
        err = np.linalg.norm(got[:, sl] - want[:, sl], axis=1)
        bound = RTOL * np.linalg.norm(want[:, sl], axis=1) + FLOOR * norm_m
        with np.errstate(divide='ignore', invalid='ignore'):
            out[:, b] = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return out


def blocks_pass(got, want, Do, Da, hidden):
    return bool(np.all(block_ratios(got, want, Do, Da, hidden) <= 1.0))


def assert_blocks(what, got, want, Do, Da, hidden):
    r = block_ratios(got, want, Do, Da, hidden)
    if np.all(r <= 1.0):
        return
    m, b = np.unravel_index(np.argmax(r), r.shape)
    sl = _block_slices(Do, Da, hidden)[b]
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    bad = [(int(mm), BLOCKS[bb]) for mm, bb in zip(*np.nonzero(r > 1.0))]
    raise AssertionError('%s: %d (task, block) pairs over the bar, e.g. %s; worst task %d block %s: |err| %.3g, |want_mb| %.3g, '
                         '|want_m| %.3g (%.2fx the bound)' % (what, len(bad), bad[:8], m, BLOCKS[b],
                                                             np.linalg.norm(got[m, sl] - want[m, sl]),
                                                             np.linalg.norm(want[m, sl]), np.linalg.norm(want[m]), r[m, b]))


# ------------------------------------------------------------------------------------------------------------ cases
class Case(object):
    """float32 inputs of one launch; theta [M, P_logical] (per task) or shared [P_logical]; old_ls [M,Da] or [M,N,Da]."""

    def __init__(self, Do, Da, hidden, M, N, seed, shared=False, ls=None, obs_scale=1.0, ls_per_sample=False,
                 n_valid=None, min_log_std=DEFAULT_MIN_LOG_STD):
        rng = np.random.RandomState(seed)
        self.Do, self.Da, self.hidden, self.M, self.N = Do, Da, hidden, M, N
        self.dims = _dims(Do, Da, hidden)
        self.shared, self.ls_per_sample, self.min_log_std = shared, ls_per_sample, min_log_std
        self.n_valid = None if n_valid is None else [int(n) for n in n_valid]
        PL = th.num_params(*self.dims)
        self.ls_lo = PL - Da
        base = th.init_params(*self.dims, rng=rng).astype(np.float64) + 0.1 * rng.randn(PL)
        theta = np.repeat(base[None], M, 0) if shared else base[None] + 0.05 * rng.randn(M, PL)
        if ls is None:
            ls = rng.uniform(-0.7, 0.3, size=Da)[None] + (0.0 if shared else 0.05 * rng.randn(M, Da))
        theta[:, self.ls_lo:] = ls
        self.theta_tasks = theta.astype(np.float32)                       # [M, PL]
        obs = rng.randn(M, N, Do) * obs_scale
        with torch.no_grad():
            mean, _ = th.dist_info(torch.from_numpy(self.theta_tasks).double(), torch.from_numpy(obs.astype(np.float32)).double(),
                                   self.dims)
        ls_eval = np.maximum(self.theta_tasks[:, self.ls_lo:].astype(np.float64), min_log_std)
        old_mean = mean.numpy() + 0.2 * rng.randn(M, N, Da)
        old_ls = (ls_eval + 0.1 * rng.randn(M, Da))[:, None, :] + (0.1 * rng.randn(M, N, Da) if ls_per_sample else 0.0)
        old_ls = np.broadcast_to(old_ls, (M, N, Da))
        act = old_mean + np.exp(old_ls) * rng.randn(M, N, Da)
        adv = rng.randn(M, N)
        f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
        self.obs, self.act, self.adv, self.old_mean = f32(obs), f32(act), f32(adv), f32(old_mean)
        self.old_ls_full = f32(old_ls)
        self.old_ls = self.old_ls_full if ls_per_sample else f32(self.old_ls_full[:, 0])
        self._nudge_clip_ties()

    @property
    def theta(self):
        return self.theta_tasks[0] if self.shared else self.theta_tasks

    @property
    def clipped(self):
        """[M, Da] bool: log_std components below min_log_std (the clip binds there when clip_log_std = 1)."""
        return self.theta_tasks[:, self.ls_lo:] < np.float32(self.min_log_std)

    def data(self, dtype=torch.float64):
        t = lambda a: torch.from_numpy(np.array(a)).to(dtype)
        return dict(obs=t(self.obs), act=t(self.act), adv=t(self.adv), mean=t(self.old_mean), log_std=t(self.old_ls_full))

    def theta_t(self, dtype=torch.float64):
        return torch.from_numpy(self.theta_tasks.copy()).to(dtype)

    def _nudge_clip_ties(self):
        """A sample whose float64 ratio lies within 1e-5 of 1 +- CLIP_EPS could take different branches of the clipped
        objective in float32 and float64: give it a zero advantage, so that both branches agree."""
        with torch.no_grad():
            mean, ls = th.dist_info(self.theta_t(), self.data()['obs'], self.dims, self.min_log_std)
            d = self.data()
            r = th.likelihood_ratio(d['act'], d['mean'], d['log_std'], mean, ls).numpy()
        tie = (np.abs(r - (1 - CLIP_EPS)) < 1e-5) | (np.abs(r - (1 + CLIP_EPS)) < 1e-5)
        self.adv[tie] = 0.0

    # oracle entry points (float64 unless dtype says otherwise)
    def grad(self, kind, obj_scale=1.0, kl_coeff=0.0, clip=True, dtype=torch.float64, **kw):
        args = (self.dims, kind, obj_scale, CLIP_EPS, kl_coeff, self.min_log_std if clip else None)
        if self.n_valid is not None:
            return oracle_ragged(oracle_grad, self.theta_t(dtype), self.data(dtype), self.n_valid, *args, **kw)
        return oracle_grad(self.theta_t(dtype), self.data(dtype), *args, **kw)

    def hvp_delta(self, kind, vec, inner_lr, kl_coeff, clip=True, dtype=torch.float64, **kw):
        vec = torch.as_tensor(vec).to(dtype)
        args = (self.dims, kind)
        rest = (inner_lr, kl_coeff, self.min_log_std if clip else None)
        if self.n_valid is not None:
            outs = []
            for m, n in enumerate(self.n_valid):
                dm = {k: v[m:m + 1, :n] for k, v in self.data(dtype).items()}
                outs.append(oracle_hvp_delta(self.theta_t(dtype)[m:m + 1], dm, *args, vec[m:m + 1], *rest, **kw))
            return torch.cat(outs, 0)
        return oracle_hvp_delta(self.theta_t(dtype), self.data(dtype), *args, vec, *rest, **kw)

    def vec(self, seed=5):
        """A random direction [M, P_logical] whose blocks have the size of the blocks of an outer gradient, as the vector the
        meta-gradient chain hands the HVP does.  (out = vec + delta is rounded to float32, so an error of ~1e-7 |vec_mb| in
        out - vec is unavoidable; with a unit-size vec it would dominate the W1 block, where H vec is small.)"""
        g = self.grad('clip', kl_coeff=0.2)[0].numpy()
        v = np.random.RandomState(seed).randn(*g.shape)
        for sl in _block_slices(self.Do, self.Da, self.hidden):
            v[:, sl] *= np.sqrt(np.mean(g[:, sl] ** 2, axis=1, keepdims=True)) + 1e-3
        return v.astype(np.float32)


def _binding_ls(M, Da, min_log_std, seed):
    """log_std [M, Da] with components on both sides of min_log_std, each at least 0.05 away from it: even components
    (odd ones on odd tasks when Da = 1) below, the others above."""
    rng = np.random.RandomState(seed)
    ls = np.empty((M, Da))
    for m in range(M):
        for d in range(Da):
            below = (d + (m if Da == 1 else 0)) % 2 == 0
            ls[m, d] = min_log_std - 0.05 - rng.uniform(0, 0.3) if below else min_log_std + 0.05 + rng.uniform(0, 0.4)
    return ls


# ---------------------------------------------------------------------------------------------------------------- CPU
def _central_difference_hvp(case, kind, vec, eps=1e-6):
    """-inner_lr H vec by central differences of the float64 oracle gradient (inner_lr = 1, no KL term)."""
    t = case.theta_t()
    v = torch.from_numpy(vec).double()
    d = case.data()
    gp, _, _ = oracle_grad(t + eps * v, d, case.dims, kind, min_log_std=case.min_log_std)
    gm, _, _ = oracle_grad(t - eps * v, d, case.dims, kind, min_log_std=case.min_log_std)
    return -(gp - gm) / (2 * eps)


@pytest.mark.parametrize('binding', [False, True], ids=['clip-free', 'clip-binding'])
@pytest.mark.parametrize('kind', ['ratio', 'loglik'])
def test_hvp_oracle_matches_central_differences(kind, binding):
    M, Da = 3, 3
    min_ls = -0.3 if binding else DEFAULT_MIN_LOG_STD
    case = Case(5, Da, 32, M, 200, seed=21, ls=_binding_ls(M, Da, min_ls, 3) if binding else None, min_log_std=min_ls)
    assert case.clipped.any() == binding and not case.clipped.all()
    vec = case.vec()
    want = case.hvp_delta(kind, vec, 1.0, 0.0).numpy()
    fd = _central_difference_hvp(case, kind, vec).numpy()
    # the finite difference carries ~1e-10 / eps of round-off: well inside the bar, and still per block
    assert_blocks('central differences', fd, want, 5, Da, 32)
    if binding:
        ls = slice(case.ls_lo, case.ls_lo + Da)
        assert np.all(want[:, ls][case.clipped] == 0.0)


# every shape of the GPU cases, with the features the bar has to hold for
CALIBRATION = [(Do, Da, h) for (Do, Da) in EXACT_SHAPES + BUCKET_SHAPES for h in (64, 32)]


@pytest.mark.parametrize('Do,Da,hidden', CALIBRATION, ids=['%dx%d-h%d' % c for c in CALIBRATION])
def test_float32_oracle_passes_with_margin(Do, Da, hidden):
    """The same oracle evaluated in float32 is a kernel with ordinary float32 round-off: it must pass the bar with a 10x
    margin on every case shape (gradients of every objective kind, the HVP delta after rounding out = vec + delta to float32,
    a binding clip, a per-sample old log_std, saturated tanh, shared parameters)."""
    M, N = 3, 257
    min_ls = -0.3
    cases = [Case(Do, Da, hidden, M, N, seed=31),
             Case(Do, Da, hidden, M, N, seed=32, ls=_binding_ls(M, Da, min_ls, 4), min_log_std=min_ls, ls_per_sample=True),
             Case(Do, Da, hidden, M, N, seed=33, obs_scale=5.0, shared=True)]
    worst = 0.0
    for case in cases:
        for kind, kl_coeff in (('ratio', 0.0), ('ratio', 0.2), ('loglik', 0.2), ('clip', 0.0), ('clip', 0.2), ('none', 1.0)):
            want, st64, _ = case.grad(kind, kl_coeff=kl_coeff)
            got, st32, _ = case.grad(kind, kl_coeff=kl_coeff, dtype=torch.float32)
            worst = max(worst, block_ratios(got.double().numpy(), want.numpy(), Do, Da, hidden).max())
        vec = case.vec()
        for kind in ('ratio', 'loglik'):
            want = case.hvp_delta(kind, vec, 0.1, 5e-4).numpy()
            d32 = case.hvp_delta(kind, vec, 0.1, 5e-4, dtype=torch.float32).numpy()
            out32 = (vec + d32).astype(np.float32)
            got = out32.astype(np.float64) - vec.astype(np.float64)
            worst = max(worst, block_ratios(got, want, Do, Da, hidden).max())
    print('float32 oracle %dx%d h%d: worst block error %.3g of the bound (margin %.1fx)' % (Do, Da, hidden, worst, 1 / worst))
    assert worst <= 0.1, worst


def _teeth_case(**kw):
    M = 3
    return Case(kw.pop('Do', 4), kw.pop('Da', 2), 64, M, kw.pop('N', 257), seed=kw.pop('seed', 41), **kw)


def test_bar_rejects_log_std_gradient_of_one_task_off_by_3e_4():
    case = _teeth_case()
    want = case.grad('ratio', kl_coeff=0.2)[0].numpy()
    got = want.copy()
    got[1, case.ls_lo:] *= 1 + 3e-4
    assert blocks_pass(want, want, case.Do, case.Da, 64)
    assert not blocks_pass(got, want, case.Do, case.Da, 64)


def test_bar_rejects_one_b2_component_off_by_3e_4():
    """Action size 1 and saturated tanh units (obs x 5), so that b2 carries a visible share of the task's gradient."""
    case = _teeth_case(Do=1, Da=1, obs_scale=5.0, ls=np.array([-1.5]))
    want = case.grad('ratio')[0].numpy()
    b2 = _block_slices(1, 1, 64)[5]
    got = want.copy()
    got[0, b2.start] *= 1 + 3e-4
    assert not blocks_pass(got, want, 1, 1, 64)


@pytest.mark.parametrize('tile', [64, 128])
def test_bar_rejects_dropping_the_last_partial_tile_of_one_task(tile):
    """257 samples: the last 64- or 128-sample tile holds one sample.  The perturbed result is the oracle on the task's
    first 256 samples."""
    case = _teeth_case(N=257)
    want = case.grad('clip', kl_coeff=0.2)[0].numpy()
    case.n_valid = [257, 257 - (257 % tile), 257]
    got = case.grad('clip', kl_coeff=0.2)[0].numpy()
    assert not blocks_pass(got, want, case.Do, case.Da, 64)
    vec = case.vec()
    case.n_valid = None
    want = case.hvp_delta('ratio', vec, 0.1, 5e-4).numpy()
    case.n_valid = [257, 257 - (257 % tile), 257]
    got = case.hvp_delta('ratio', vec, 0.1, 5e-4).numpy()
    assert not blocks_pass(got, want, case.Do, case.Da, 64)


def test_bar_rejects_two_tasks_swapped():
    case = _teeth_case()
    want = case.grad('ratio')[0].numpy()
    got = want[[1, 0, 2]]
    assert not blocks_pass(got, want, case.Do, case.Da, 64)


def test_bar_rejects_a_missing_clip_mask():
    min_ls = -0.3
    case = _teeth_case(Da=2, ls=_binding_ls(3, 2, min_ls, 6), min_log_std=min_ls)
    assert case.clipped.any()
    want = case.grad('ratio', kl_coeff=0.2)[0].numpy()
    got = case.grad('ratio', kl_coeff=0.2, straight_through_clip=True)[0].numpy()
    assert not blocks_pass(got, want, case.Do, case.Da, 64)
    vec = case.vec()
    want = case.hvp_delta('ratio', vec, 0.1, 5e-4).numpy()
    got = case.hvp_delta('ratio', vec, 0.1, 5e-4, straight_through_clip=True).numpy()
    assert not blocks_pass(got, want, case.Do, case.Da, 64)


def test_bar_rejects_ignoring_the_per_sample_old_log_std():
    case = _teeth_case(ls_per_sample=True)
    want_g = case.grad('ratio', kl_coeff=0.2)[0].numpy()
    vec = case.vec()
    want_h = case.hvp_delta('ratio', vec, 0.1, 5e-4).numpy()
    case.old_ls_full = np.ascontiguousarray(np.broadcast_to(case.old_ls_full[:, :1], case.old_ls_full.shape))
    assert not blocks_pass(case.grad('ratio', kl_coeff=0.2)[0].numpy(), want_g, case.Do, case.Da, 64)
    assert not blocks_pass(case.hvp_delta('ratio', vec, 0.1, 5e-4).numpy(), want_h, case.Do, case.Da, 64)


def test_bar_rejects_a_missing_kl_term_in_the_hvp():
    """ProMP's initial inner-KL coefficient, 5e-4."""
    case = _teeth_case()
    vec = case.vec()
    want = case.hvp_delta('ratio', vec, 0.1, 5e-4).numpy()
    got = case.hvp_delta('ratio', vec, 0.1, 0.0).numpy()
    assert not blocks_pass(got, want, case.Do, case.Da, 64)


def plan_tiles(M, N, slots, tb=128):
    """Python copy of plan_tiles (csrc/policy.cu): (ntiles, grid, q, kmax) of the one-wave persistent tile plan."""
    ntiles = -(-N // tb)
    T = M * ntiles
    g = max(1, min(T, slots))
    q = -(-T // g)
    return ntiles, -(-T // q), q, -(-q // ntiles) + 1


def test_plan_tiles_copy_gives_the_geometries_the_gpu_cases_name():
    # 132 SMs (H100 SXM), one tensor-core CTA per SM
    assert plan_tiles(1, 40000, 132) == (313, 105, 3, 2)
    assert plan_tiles(300, 100, 132) == (1, 100, 3, 4)
    assert plan_tiles(40, 2000, 132) == (16, 128, 5, 2)
    assert plan_tiles(96, 1000, 132) == (8, 128, 6, 2)
    assert plan_tiles(7, 2000, 132) == (16, 112, 1, 2)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')


def _policy(case):
    from promp_b200.policies import MetaGaussianMLPPolicy
    pol = MetaGaussianMLPPolicy(name='p', obs_dim=case.Do, action_dim=case.Da, meta_batch_size=case.M,
                                hidden_sizes=(case.hidden, case.hidden))
    assert pol.num_params_logical == case.theta_tasks.shape[1]
    return pol


def _caps(Do, Da):
    if (Do, Da) in EXACT_SHAPES:
        return Do, Da
    return (8 if Do <= 8 else 20), (2 if Da <= 2 else 8)


PATHS = ('cuda', 'tc256', 'tc512', 'h32')


@contextlib.contextmanager
def _path(path):
    from promp_b200 import _lib
    try:
        _lib.set_option('tensor_cores', 0 if path == 'cuda' else 1)
        _lib.set_option('tc_threads', dict(tc256=256, tc512=512).get(path, 0))
        yield
    finally:
        _lib.set_option('tensor_cores', 1)
        _lib.set_option('tc_threads', 0)
        _lib.set_option('chain', -1)


def _expected_kernels(path, Do, Da, hidden):
    """Names (template arguments included) of the gradient and HVP kernels a path must run."""
    cd, ca = _caps(Do, Da)
    if hidden == 32 or path == 'cuda':
        return ['policy_grad_kernel<%d,%d,%d>' % (cd, ca, hidden), 'policy_hvp_kernel<%d,%d,%d>' % (cd, ca, hidden)]
    nq = dict(tc256=2, tc512=4).get(path, 4 if cd <= 4 else 2)
    return ['policy_grad_tc_kernel<%d,%d,%d>' % (cd, ca, nq), 'policy_hvp_tc_kernel<%d,%d,%d>' % (cd, ca, nq)]


class Launcher(object):
    """The case's inputs on the device and the C entry points of its policy (`policy.entries`)."""

    def __init__(self, case):
        from promp_b200 import _lib
        self.lib, self.case = _lib, case
        self.pol = pol = _policy(case)
        self.P = pol.num_params
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.params = dev(pol.pad_flat(case.theta))
        self.stride = 0 if case.shared else self.P
        obs, act, adv, mean = case.obs.copy(), case.act.copy(), case.adv.copy(), case.old_mean.copy()
        if case.n_valid is not None:         # poison in the padding rows (test_policy_dims._ragged_phase)
            for m, n in enumerate(case.n_valid):
                obs[m, n:] = 1e3; act[m, n:] = -50.0; adv[m, n:] = 1e4; mean[m, n:] = 7.0
        self.obs, self.act, self.adv, self.mean, self.old_ls = dev(obs), dev(act), dev(adv), dev(mean), dev(case.old_ls)
        self.n_valid = None if case.n_valid is None else torch.tensor(case.n_valid, dtype=torch.int32, device='cuda')
        need = getattr(_lib.load(), pol.entries['workspace_bytes'])(case.M, case.N, case.Do, case.Da, pol.hidden)
        self.ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device='cuda')

    def logical(self, t):
        return self.pol.unpad_flat(t.cpu().numpy())

    def pads(self, t):
        mask = np.ones(self.P, dtype=bool)
        mask[self.pol._pad_index_np] = False
        return t.cpu().numpy()[:, mask]

    def grad(self, kind, obj_scale=1.0, kl_coeff=0.0, clip=1, sgd_lr=0.1):
        c, M = self.case, self.case.M
        grad = torch.full((M, self.P), float('nan'), device='cuda')
        newp = torch.full((M, self.P), float('nan'), device='cuda')
        stats = torch.full((M, 4), float('nan'), device='cuda')
        p = self.lib.ptr
        self.lib.call(self.pol.entries['grad_ex'], c.Do, c.Da, self.pol.hidden, M, c.N, p(self.n_valid), p(self.params),
                      self.stride, p(self.obs), p(self.act), p(self.adv), p(self.mean), p(self.old_ls), int(c.ls_per_sample),
                      OBJ[kind], float(obj_scale), CLIP_EPS, float(kl_coeff), int(clip), float(c.min_log_std), p(grad), p(newp),
                      float(sgd_lr), p(stats), None, None, None, None, p(self.ws), self.ws.numel() * 4, self.lib.stream())
        torch.cuda.synchronize()
        return grad, newp, stats

    def hvp(self, kind, vec, inner_lr=0.1, kl_coeff=5e-4, clip=1):
        c, M = self.case, self.case.M
        v = torch.from_numpy(self.pol.pad_flat(vec)).cuda()
        out = torch.full((M, self.P), float('nan'), device='cuda')
        stats = torch.full((M, 4), float('nan'), device='cuda')
        p = self.lib.ptr
        self.lib.call(self.pol.entries['hvp_ragged'], c.Do, c.Da, self.pol.hidden, M, c.N, p(self.n_valid), p(self.params),
                      self.stride, p(self.obs), p(self.act), p(self.adv), p(self.mean), p(self.old_ls), int(c.ls_per_sample),
                      OBJ[kind], float(inner_lr), float(kl_coeff), int(clip), float(c.min_log_std), p(v), p(out), p(stats),
                      p(self.ws), self.ws.numel() * 4, self.lib.stream())
        torch.cuda.synchronize()
        return v, out, stats


def check_grad(L, what, kind, obj_scale=1.0, kl_coeff=0.0, clip=1, sgd_lr=0.1):
    """One gradient launch against the oracle: blocks, stats, pads, clipped components, out_params."""
    c = L.case
    grad, newp, stats = L.grad(kind, obj_scale, kl_coeff, clip, sgd_lr)
    want, st_want, st_scale = c.grad(kind, obj_scale, kl_coeff, clip=bool(clip))
    g = L.logical(grad)
    assert np.all(L.pads(grad) == 0.0), what + ': pad entries of the gradient are not 0.0'
    if clip:
        assert np.all(g[:, c.ls_lo:][c.clipped] == 0.0), what + ': clipped log_std components have a gradient'
    assert_blocks(what + ' gradient', g, want.numpy(), c.Do, c.Da, c.hidden)
    st = stats.cpu().numpy()[:, :3].astype(np.float64)
    bound = RTOL * np.abs(st_want.numpy()) + 1e-6 * st_scale.numpy()
    assert np.all(np.abs(st - st_want.numpy()) <= bound), (what + ' stats', st, st_want.numpy())
    # out_params = params - sgd_lr * grad with the kernel's own gradient, to one ulp of the operands (a fused multiply-add
    # rounds once, a multiply then subtract twice)
    prm = L.params.view(-1, L.P).expand(c.M, -1).cpu().numpy()
    step = np.float32(sgd_lr) * grad.cpu().numpy().astype(np.float64)
    exact = prm.astype(np.float64) - step
    ulp = np.spacing(np.maximum(np.abs(prm), np.abs(step).astype(np.float32)))
    assert np.all(np.abs(newp.cpu().numpy() - exact) <= ulp), what + ': out_params'
    return g


def check_hvp(L, what, kind, inner_lr=0.1, kl_coeff=5e-4, clip=1):
    c = L.case
    vec = c.vec()
    v, out, stats = L.hvp(kind, vec, inner_lr, kl_coeff, clip)
    want = c.hvp_delta(kind, vec, inner_lr, kl_coeff, clip=bool(clip)).numpy()
    out_np = out.cpu().numpy()
    assert np.all(L.pads(out) == L.pads(v)), what + ': out != vec on pad entries'
    delta = L.pol.unpad_flat(out_np).astype(np.float64) - vec.astype(np.float64)
    if clip:
        assert np.all(delta[:, c.ls_lo:][c.clipped] == 0.0), what + ': out != vec on clipped log_std components'
    assert_blocks(what + ' HVP (out - vec)', delta, want, c.Do, c.Da, c.hidden)
    _, st_want, st_scale = c.grad(kind, clip=bool(clip))
    st = stats.cpu().numpy()[:, :2].astype(np.float64)
    bound = RTOL * np.abs(st_want.numpy()[:, :2]) + 1e-6 * st_scale.numpy()[:, :2]
    assert np.all(np.abs(st - st_want.numpy()[:, :2]) <= bound), (what + ' HVP stats', st, st_want.numpy()[:, :2])


def _kernels_run_by(fn):
    """Names (whitespace removed) of the CUDA kernels `fn` launches, from torch.profiler; None without CUPTI."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device='cuda').add_(1)      # a first kernel, so that the session is running before the launches of fn
        fn()
        torch.cuda.synchronize()
    names = [re.sub(r'\s+', '', e.name) for e in prof.events()]
    return names or None


# Observation prefetch of the tensor-core tile loops (XPRE in grad_tc_tiles / hvp_tc_tiles): on when a 128-sample tile of
# observations is one or two floats per thread and DA <= 2.  Per (obs cap, act cap): 256 threads / 512 threads.
#   (2,2) (4,2): prefetch / prefetch      (1,1) -> (8,2): no prefetch / prefetch
#   (17,6), (5,3) -> (8,8), (19,8) -> (20,8): no prefetch / no prefetch
SHAPES = EXACT_SHAPES + BUCKET_SHAPES


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da', SHAPES, ids=['%dx%d' % s for s in SHAPES])
@pytest.mark.parametrize('path', PATHS)
def test_paths_and_shapes(path, Do, Da):
    """Every kernel path (CUDA cores, tensor cores at 256 and 512 threads, hidden 32) at every exact and bucket shape;
    the profiler confirms which kernel ran (a tensor-core case must not quietly run the CUDA-core kernel)."""
    _cuda()
    hidden = 32 if path == 'h32' else 64
    case = Case(Do, Da, hidden, 3, 300, seed=100 + Do * 10 + Da)
    with _path(path):
        L = Launcher(case)
        check_grad(L, '%s %dx%d' % (path, Do, Da), 'ratio', kl_coeff=0.1)
        check_hvp(L, '%s %dx%d' % (path, Do, Da), 'ratio')
        names = _kernels_run_by(lambda: (L.grad('ratio'), L.hvp('ratio', case.vec())))
    if names is None:        # no CUDA activity recorded: CUPTI is not available, nothing to assert
        return
    print('%s %dx%d ran %s' % (path, Do, Da, sorted(set(k for k in names if 'policy_' in k))))
    for name in _expected_kernels(path, Do, Da, hidden):
        assert any(name in k for k in names), (name, sorted(set(names)))


# (path, shape): CUDA cores (64-sample tiles); tensor cores (128-sample tiles) with and without the observation prefetch
EDGE_CONFIGS = [('cuda', (5, 3)), ('tc512', (2, 2)), ('tc256', (17, 6))]


@pytest.mark.gpu
@pytest.mark.parametrize('N', TILE_EDGE_N)
@pytest.mark.parametrize('path,shape', EDGE_CONFIGS, ids=['cuda-5x3', 'tc-prefetch-2x2', 'tc-noprefetch-17x6'])
def test_tile_edges(path, shape, N):
    _cuda()
    Do, Da = shape
    case = Case(Do, Da, 64, 2, N, seed=200 + N)
    with _path(path):
        L = Launcher(case)
        check_grad(L, '%s N=%d' % (path, N), 'clip', kl_coeff=0.1)
        check_hvp(L, '%s N=%d' % (path, N), 'loglik')


# Persistent multi-tile geometries of the tensor-core kernels (per-task parameters, param_stride = P).  ntiles / grid / q /
# kmax from plan_tiles with 132 SMs and one CTA per SM (checked below against the device's SM count):
GEOMETRIES = [
    (2, 2, 1, 40000),     # one task over many CTAs: ntiles 313, grid 105, q 3, kmax 2 (next-tile observation prefetch)
    (4, 2, 300, 100),     # several whole tasks per CTA: ntiles 1, grid 100, q 3, kmax 4 (weight reload inside a CTA)
    (2, 2, 40, 2000),     # the benchmark shape: ntiles 16, grid 128, q 5, kmax 2
    (17, 6, 96, 1000),    # tasks straddling CTAs: ntiles 8, grid 128, q 6, kmax 2 (no prefetch)
]


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,M,N', GEOMETRIES, ids=['1x40000', '300x100', '40x2000', '96x1000-17x6'])
def test_scheduling_geometry(Do, Da, M, N):
    _cuda()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ntiles, grid, q, kmax = plan_tiles(M, N, sms)
    assert q > 1, 'the geometry must give each CTA several tiles'
    if M > 1 and ntiles == 1:
        assert kmax > 2
    case = Case(Do, Da, 64, M, N, seed=300 + M)
    with _path('tc'):
        L = Launcher(case)
        check_grad(L, 'geometry %dx%d' % (M, N), 'ratio', kl_coeff=0.1)
        check_hvp(L, 'geometry %dx%d' % (M, N), 'ratio')


KINDS = [('ratio', 0.0), ('ratio', 0.2), ('loglik', 0.0), ('loglik', 0.2), ('clip', 0.0), ('clip', 0.2), ('none', 0.0),
         ('none', 1.0)]


@pytest.mark.gpu
@pytest.mark.parametrize('shared', [True, False], ids=['shared-theta', 'per-task-theta'])
@pytest.mark.parametrize('kind,kl_coeff', KINDS, ids=['%s-kl%g' % k for k in KINDS])
def test_objective_kinds(kind, kl_coeff, shared):
    """Every objective kind with and without the KL term (NONE with kl_coeff = 1 is TRPO's constraint gradient); the HVP
    for the two inner objectives.  obj_scale != 1 checks that it scales the surrogate only."""
    _cuda()
    case = Case(4, 2, 64, 5, 700, seed=400, shared=shared)
    with _path('tc'):
        L = Launcher(case)
        check_grad(L, '%s kl %g' % (kind, kl_coeff), kind, obj_scale=0.7, kl_coeff=kl_coeff)
        if kind in ('ratio', 'loglik'):
            check_hvp(L, '%s kl %g' % (kind, kl_coeff), kind, kl_coeff=kl_coeff)


FEATURE_PATHS = [('cuda', (5, 3), 64), ('tc256', (17, 6), 64), ('tc512', (2, 2), 64), ('h32', (19, 8), 32)]
FEATURE_IDS = ['cuda-5x3', 'tc256-17x6', 'tc512-2x2', 'h32-19x8']


@pytest.mark.gpu
@pytest.mark.parametrize('path,shape,hidden', FEATURE_PATHS, ids=FEATURE_IDS)
def test_binding_log_std_clip(path, shape, hidden):
    """min_log_std between the log_std components: the clipped ones get no gradient and out == vec, the others do."""
    _cuda()
    Do, Da = shape
    M, min_ls = 4, -0.3
    case = Case(Do, Da, hidden, M, 333, seed=500, ls=_binding_ls(M, Da, min_ls, 7), min_log_std=min_ls)
    assert case.clipped.any() and not case.clipped.all()
    with _path(path):
        L = Launcher(case)
        for kind in ('ratio', 'loglik'):
            check_grad(L, 'clip %s' % kind, kind, kl_coeff=0.2)
            check_hvp(L, 'clip %s' % kind, kind, kl_coeff=0.01)
        check_grad(L, 'clip outer', 'clip', kl_coeff=0.2)


@pytest.mark.gpu
@pytest.mark.parametrize('path,shape,hidden', FEATURE_PATHS, ids=FEATURE_IDS)
def test_old_log_std_per_sample(path, shape, hidden):
    """ls_per_sample = 1 (reference-style sample dicts) with an old log_std that varies over samples and tasks."""
    _cuda()
    Do, Da = shape
    case = Case(Do, Da, hidden, 3, 300, seed=600, ls_per_sample=True)
    assert np.ptp(case.old_ls, axis=1).min() > 0
    with _path(path):
        L = Launcher(case)
        check_grad(L, 'ls_per_sample', 'ratio', kl_coeff=0.2)
        check_hvp(L, 'ls_per_sample', 'ratio')


@pytest.mark.gpu
@pytest.mark.parametrize('path,shape,hidden', FEATURE_PATHS, ids=FEATURE_IDS)
def test_ragged_n_valid(path, shape, hidden):
    """n_valid of 1, 64, 127, 128, 129 and N; rows past n_valid hold poison."""
    _cuda()
    Do, Da = shape
    N = 300
    case = Case(Do, Da, hidden, 6, N, seed=700, n_valid=[1, 64, 127, 128, 129, N])
    with _path(path):
        L = Launcher(case)
        check_grad(L, 'ragged', 'clip', kl_coeff=0.2)
        check_grad(L, 'ragged', 'ratio')
        check_hvp(L, 'ragged', 'ratio')


@pytest.mark.gpu
@pytest.mark.parametrize('path,shape,hidden', FEATURE_PATHS, ids=FEATURE_IDS)
def test_saturated_tanh(path, shape, hidden):
    """Observations x 5 drive the hidden tanh units deep into saturation."""
    _cuda()
    Do, Da = shape
    case = Case(Do, Da, hidden, 3, 300, seed=800, obs_scale=5.0)
    with _path(path):
        L = Launcher(case)
        check_grad(L, 'saturated', 'ratio', kl_coeff=0.2)
        check_hvp(L, 'saturated', 'loglik')


FORWARD = [('exact', (17, 6), 64), ('exact', (2, 2), 32), ('padded', (5, 3), 64), ('padded', (19, 8), 32)]


@pytest.mark.gpu
@pytest.mark.parametrize('N', TILE_EDGE_N)
@pytest.mark.parametrize('entry,shape,hidden', FORWARD, ids=['%s-%dx%d-h%d' % (e, s[0], s[1], h) for e, s, h in FORWARD])
def test_forward(entry, shape, hidden, N):
    """promp_policy_forward (exact table) and promp_policy_forward_padded against dist_info, shared and per-task parameters."""
    _cuda()
    from promp_b200 import _lib
    Do, Da = shape
    for shared in (True, False):
        case = Case(Do, Da, hidden, 3, N, seed=900 + N, shared=shared)
        pol = _policy(case)
        assert pol.entries['forward'] == ('promp_policy_forward' + ('_padded' if entry == 'padded' else ''))
        params = torch.from_numpy(pol.pad_flat(case.theta)).cuda()
        obs = torch.from_numpy(case.obs).cuda()
        mean = torch.full((case.M, N, Da), float('nan'), device='cuda')
        _lib.call(pol.entries['forward'], Do, Da, hidden, case.M, N, _lib.ptr(params), 0 if shared else pol.num_params,
                  _lib.ptr(obs), _lib.ptr(mean), _lib.stream())
        with torch.no_grad():
            want, _ = th.dist_info(case.theta_t(), case.data()['obs'], case.dims)
        got = mean.cpu().numpy().astype(np.float64)
        want = want.numpy()
        for m in range(case.M):
            err = np.linalg.norm(got[m] - want[m])
            assert err <= 1e-5 * np.linalg.norm(want[m]) + 1e-7 * math.sqrt(want[m].size), (m, err)


# ---- the production meta-gradient ------------------------------------------------------------------------------------
def _promp_setup(Do, Da, M, N, min_std, seed):
    """A ProMP algorithm on a policy whose min_std binds on some log_std components, and two phases of float32 data."""
    from promp_b200.meta_algos import ProMP
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers.device_data import PhaseData
    np.random.seed(seed)
    pol = MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64), min_std=min_std)
    min_ls = pol.min_log_std
    case = Case(Do, Da, 64, 1, 1, seed=seed, shared=True, ls=_binding_ls(1, Da, min_ls, seed)[0], min_log_std=min_ls)
    th_l = case.theta
    pol.set_params(th_l)
    algo = ProMP(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=1,
                 clip_eps=CLIP_EPS, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    dims = _dims(Do, Da, 64)
    cpus, phases = [], []
    theta_s = torch.from_numpy(th_l).double().view(1, -1).expand(M, -1)
    for s in range(2):
        rng = np.random.RandomState(seed + 1 + s)
        obs = torch.from_numpy(rng.randn(M, N, Do).astype(np.float32)).double()
        with torch.no_grad():
            mean, ls = th.dist_info(theta_s, obs, dims, min_ls)
        old_mean = (mean + 0.1 * torch.from_numpy(rng.randn(M, N, Da))).float().double()
        old_ls = (ls + 0.05 * torch.from_numpy(rng.randn(M, 1, Da))).float().double().expand(M, N, Da)
        act = (old_mean + torch.exp(old_ls) * torch.from_numpy(rng.randn(M, N, Da))).float().double()
        adv = torch.from_numpy(rng.randn(M, N).astype(np.float32)).double()
        cpus.append(dict(obs=obs, act=act, adv=adv, mean=old_mean, log_std=old_ls.contiguous()))
        if s == 0:      # the adapted parameters (step-0 graph: clipped log_std) give the outer phase's ratios
            t = theta_s.clone().requires_grad_(True)
            theta_s = th.adapt_sym(t, cpus[0], dims, 0.1, min_log_std=min_ls)[0].detach()
    with torch.no_grad():
        mean, ls = th.dist_info(theta_s, cpus[1]['obs'], dims)
        r = th.likelihood_ratio(cpus[1]['act'], cpus[1]['mean'], cpus[1]['log_std'], mean, ls)
    cpus[1]['adv'][(torch.abs(r - (1 - CLIP_EPS)) < 1e-5) | (torch.abs(r - (1 + CLIP_EPS)) < 1e-5)] = 0.0
    for c in cpus:
        ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
        ph.obs.copy_(c['obs']); ph.act.copy_(c['act']); ph.mean.copy_(c['mean']); ph.log_std.copy_(c['log_std'][:, 0])
        ph.adv = c['adv'].float().cuda()
        phases.append(ph)
    return pol, algo, case, cpus, phases


def _meta_grad_tasks(case, cpus, coeff, min_ls):
    out, objs = [], []
    for m in range(cpus[0]['obs'].shape[0]):
        t64 = torch.tensor(case.theta, dtype=torch.float64, requires_grad=True)
        data_m = [{k: v[m:m + 1] for k, v in c.items()} for c in cpus]
        obj, _, _ = th.meta_objective(t64, data_m, case.dims, 0.1, 'promp', CLIP_EPS, coeff, min_log_std=min_ls)
        out.append(torch.autograd.grad(obj, t64)[0].numpy())
        objs.append(float(obj.detach()))
    return np.stack(out), np.array(objs)


@pytest.mark.gpu
@pytest.mark.parametrize('Do,Da,M,N', [(2, 2, 40, 2000), (5, 3, 5, 129)], ids=['40x2000-2x2', '5x129-5x3'])
@pytest.mark.parametrize('chain', [0, 1])
def test_meta_gradient_per_task_with_binding_min_std(Do, Da, M, N, chain):
    """ProMP._objective_pass(reduce=False) per task against the float64 meta_objective gradient, with a min_std that clips
    some log_std components in the step-0 graph (and so in the chain's HVP stage); chain 1 = the dataflow kernel, 0 = one
    launch per stage."""
    _cuda()
    from promp_b200 import _lib
    import ctypes
    pol, algo, case, cpus, phases = _promp_setup(Do, Da, M, N, min_std=0.8, seed=1000 + N)
    assert case.clipped.any() and not case.clipped.all()
    want, _ = _meta_grad_tasks(case, cpus, list(algo.inner_kl_coeff), pol.min_log_std)
    algo.use_chain = True
    try:
        _lib.set_option('chain', chain)
        stages = (_lib.PolicyStage * 3)()
        for s, kind in enumerate((0, 0, 1)):
            stages[s].kind, stages[s].N = kind, N
        n_launch = getattr(_lib.load(), pol.entries['chain_num_launches'])(Do, Da, 64, M, 3, ctypes.cast(stages, ctypes.c_void_p))
        assert n_launch == (1 if chain else 3)
        res = algo._objective_pass(phases, want_grad=True, reduce=False)
        got = pol.unpad_flat(res['grad_tasks'].cpu().numpy())
    finally:
        _lib.set_option('chain', -1)
    mask = np.ones(pol.num_params, dtype=bool)
    mask[pol._pad_index_np] = False
    assert np.all(res['grad_tasks'].cpu().numpy()[:, mask] == 0.0)
    assert_blocks('meta-gradient chain=%d' % chain, got, want, Do, Da, 64)


@pytest.mark.gpu
def test_promp_optimize_policy_with_binding_min_std_does_not_reuse_adapt():
    """With the step-0 clip binding, the first Adam epoch's inner pass must not re-use the _adapt launch (which ran without
    the clip): the first-epoch meta-gradient (Adam's first moment / (1 - beta1)) and LossBefore match float64."""
    _cuda()
    Do, Da, M, N = 4, 2, 6, 500
    pol, algo, case, cpus, phases = _promp_setup(Do, Da, M, N, min_std=0.8, seed=1100)
    from promp_b200.samplers.device_data import SamplesData
    samples = [[SamplesData(p, m) for m in range(M)] for p in phases]
    pol.switch_to_pre_update()
    algo._adapt(samples[0])
    assert algo._adapt_cache is not None
    assert int(algo._reuse_bufs[0].item()) == 0, '_adapt must report that the step-0 clip binds'
    pol.switch_to_pre_update()
    want, objs = _meta_grad_tasks(case, cpus, list(algo.inner_kl_coeff), pol.min_log_std)
    loss_want = float(objs.mean())
    algo.optimize_policy(samples, log=False)
    g_got = pol.unpad_flat((algo.optimizer.m / (1 - 0.9)).cpu().numpy()[None])
    assert_blocks('first-epoch meta-gradient', g_got, want.mean(0, keepdims=True), Do, Da, 64)
    loss_before = algo.last_stats['loss_before']
    assert abs(loss_before - loss_want) <= RTOL * max(1.0, abs(loss_want)), (loss_before, loss_want)
