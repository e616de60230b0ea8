"""The sample-processing kernel (promp_process_samples / _ragged / promp_baseline_fit) on every launch geometry its host
code can select, against the float64 numpy oracle (oracle/numpy_half.py, pinned to the unmodified reference by
test_oracle_golden.py).

process_fused_kernel picks its code path from the shape: whether the front / finish stage keeps its sample arrays in
shared memory (<stage_f, stage_l>; otherwise the float64 workspace), whether every time step is covered by the t/100 table
(tt_cap <= 1024), whether the per-chunk path statistics go through the warp-0 reduction (EPC <= 32) or block_reduce, and
how many chunks (C) a task is split into.  promp_process_launch_info reports that choice without touching the device:

  - the CPU tests pin the geometry of every GPU case below and sweep obs_dim 1..19 over fixed and ragged shapes for the
    invariant that no shape stages the finish stage without staging the front stage;
  - the GPU tests run each case, check that it still lands on the path it is meant to hit, and compare returns, advantages,
    baseline fitted values Phi w and the per-task statistics row with the oracle.  They then run every case again in
    reverse order on the same shared workspace and require bit-identical outputs and an all-zero ticket header after
    every launch.
"""
import ctypes
import functools
from collections import OrderedDict

import numpy as np
import pytest

REG = 1e-5
GEOM_KEYS = ('C', 'EPC', 'chunk_cap', 'finish_cap', 'tt_cap', 'pred_tile', 'stage_f', 'stage_l')
TICKET_HEADER_DOUBLES = 65536 * 4 // 8        # arrival tickets at the start of the processing workspace
# baseline fitted values Phi w: relative error bar.  The oracle's own float64 spread on these systems (np.linalg.lstsq vs
# scipy.linalg.solve(assume_a='pos') of the same ridge system) is at most 3.2e-12, at H = 1500, obs_dim 17; the kernel's
# Cholesky solve was measured at most 2.9e-12 from the oracle on an H100.
FIT_BAR = 1e-9


# ------------------------------------------------------------------------------------------------------------- cases
# fixed-horizon cases: (M, E, H, obs_dim, discount, gae_lambda, normalize_adv, positive_adv)
FIXED = OrderedDict([
    ('finish_ws64_h600',    (4, 20, 600, 2, 0.99, 0.97, True, False)),
    ('finish_ws64_cheetah', (4, 60, 200, 17, 0.99, 1.0, False, False)),
    ('past_table_ws64',     (2, 12, 1100, 2, 0.99, 1.0, False, False)),
    ('past_table_staged',   (2, 1, 1500, 17, 0.995, 0.95, False, False)),
    ('wide_chunks',         (600, 40, 5, 2, 0.99, 1.0, True, False)),
    ('many_chunks',         (1, 600, 10, 2, 0.95, 0.9, True, True)),
    ('obs_dim_1',           (3, 20, 100, 1, 1.0, 0.0, True, False)),
    ('obs_dim_4',           (3, 20, 100, 4, 1.0, 0.5, False, True)),
    ('obs_dim_19',          (3, 20, 100, 19, 0.97, 0.0, False, False)),
])
RAGGED_HYPER = (0.99, 0.97, True, False)
EARLY_TERM = dict(M=3, E=40, H=200)
CASE_ORDER = list(FIXED) + ['ragged_ws64', 'early_term', 'baseline_fit']

# geometry each case is built to exercise: (stage_f, stage_l, tt_cap, EPC > 32, C); None = C follows from the inputs
WANT_GEOMETRY = {
    'finish_ws64_h600':    (1, 0, 600, False, 20),
    'finish_ws64_cheetah': (1, 0, 200, False, 60),
    'past_table_ws64':     (1, 0, 1024, False, 12),
    'past_table_staged':   (1, 1, 1024, False, 1),
    'wide_chunks':         (1, 1, 6, True, 1),
    'many_chunks':         (1, 1, 10, False, 300),
    'obs_dim_1':           (1, 1, 100, False, 20),
    'obs_dim_4':           (1, 1, 100, False, 20),
    'obs_dim_19':          (1, 1, 100, False, 20),
    'ragged_ws64':         (0, 0, 1024, False, None),
    'early_term':          (0, 0, 1024, True, 176),
    'baseline_fit':        (0, 0, 1024, False, 20),
}


def _walk(rng, L, Do):
    """float32-representable random-walk observations with ~1% entries pushed past the +-10 feature clip."""
    obs = np.cumsum(0.3 * rng.randn(L, Do), axis=0)
    far = rng.rand(L, Do) < 0.01
    obs[far] += np.where(rng.rand(int(far.sum())) < 0.5, -25.0, 25.0)
    return obs.astype(np.float32).astype(np.float64)


def _rewards(rng, L):
    """~40 % zero rewards, float32-representable."""
    return (rng.randn(L) * (rng.rand(L) < 0.6)).astype(np.float32).astype(np.float64)


def _path(rng, L, Do):
    return dict(observations=_walk(rng, L, Do), rewards=_rewards(rng, L))


@functools.lru_cache(maxsize=None)
def host_inputs(name):
    """Seeded host paths of a case: list (tasks) of lists of {observations, rewards} (float64 holding float32 values)."""
    rng = np.random.RandomState(sum(map(ord, name)))
    if name in FIXED:
        M, E, H, Do = FIXED[name][:4]
        return [[_path(rng, H, Do) for _ in range(E)] for _ in range(M)]
    if name == 'ragged_ws64':
        # two tasks of ~15 000 samples, paths of 1 .. 1500 steps (some past the 1024-step time table)
        tasks = []
        for extra in ([1, 1500, 1200, 2, 1030], [1500, 1, 1, 700, 1100]):
            lens = list(extra)
            while sum(lens) < 14000:
                lens.append(int(rng.randint(1, 1501)))
            rng.shuffle(lens)
            tasks.append([_path(rng, L, 2) for L in lens])
        return tasks
    if name == 'baseline_fit':
        lens = [1500] + [int(x) for x in rng.randint(1000, 1450, size=19)]       # 20 paths, > 20 000 samples
        paths = [_path(rng, L, 2) for L in lens]
        for p in paths:
            p['returns'] = _discount_cumsum(p['rewards'], 0.99)
        return [paths]
    raise KeyError(name)


def _discount_cumsum(x, g):
    from oracle import numpy_half as nh
    return nh.discount_cumsum(x, g)


def case_shape(name):
    """(M, max_paths, H, obs_dim, NS, ragged) exactly as the entry point of the case passes them to the geometry."""
    if name in FIXED:
        M, E, H, Do = FIXED[name][:4]
        return M, E, H, Do, E * H, 0
    if name == 'ragged_ws64':
        tasks = host_inputs(name)
        n_valid = [sum(len(p['rewards']) for p in t) for t in tasks]
        return len(tasks), max(len(t) for t in tasks), 0, 2, (max(n_valid) + 3) // 4 * 4, 1     # RaggedPhaseData layout
    if name == 'early_term':
        M, E, H = EARLY_TERM['M'], EARLY_TERM['E'], EARLY_TERM['H']
        T = 2 * H - 1                       # MetaSampler._obtain_samples_fused_early: timeline of 2H-1 steps per env slot
        return M, E * T, 0, 2, (E * T + 3) // 4 * 4, 1
    if name == 'baseline_fit':
        paths = host_inputs(name)[0]
        return 1, len(paths), 0, 2, sum(len(p['rewards']) for p in paths), 1
    raise KeyError(name)


def longest_step(name):
    if name in FIXED:
        return FIXED[name][2] - 1
    if name == 'early_term':
        return None                         # short paths (origin-seeking policy): the table covers them
    return max(len(p['rewards']) for t in host_inputs(name) for p in t) - 1


def _library():
    import __graft_entry__ as ge
    ge.build()
    from promp_b200 import _lib
    return _lib.load()


def launch_info(lib, M, max_paths, H, obs_dim, NS, ragged):
    out = (ctypes.c_int32 * 8)()
    rc = lib.promp_process_launch_info(M, max_paths, H, obs_dim, NS, int(ragged), out)
    assert rc == 0, lib.promp_last_error()
    return dict(zip(GEOM_KEYS, list(out)))


def check_geometry(lib, name):
    g = launch_info(lib, *case_shape(name))
    sf, sl, tt_cap, wide, C = WANT_GEOMETRY[name]
    assert (g['stage_f'], g['stage_l']) == (sf, sl), (name, g)
    assert g['tt_cap'] == tt_cap and (g['EPC'] > 32) == wide, (name, g)
    if C is not None:
        assert g['C'] == C, (name, g)
    else:
        assert g['C'] == case_shape(name)[1] and g['EPC'] == 1, (name, g)
    last = longest_step(name)
    if tt_cap == 1024 and last is not None:
        assert last >= g['tt_cap'], (name, last, g)          # some steps take the inline t/100 branch
    return g


# --------------------------------------------------------------------------------------------------------- CPU tests
def test_case_geometry_pins():
    """Every GPU case below lands on the path it is meant to exercise; together they reach <true,true>, <true,false>,
    <false,false>, the inline time features, block_reduce, C >= 100 and obs_dim 1, 4 and 19."""
    lib = _library()
    geoms = {name: check_geometry(lib, name) for name in CASE_ORDER}
    variants = {(g['stage_f'], g['stage_l']) for g in geoms.values()}
    assert variants == {(1, 1), (1, 0), (0, 0)}
    assert any(g['EPC'] > 32 for g in geoms.values()) and max(g['C'] for g in geoms.values()) >= 100
    assert {case_shape(n)[3] for n in CASE_ORDER} >= {1, 2, 4, 17, 19}
    past = [n for n in CASE_ORDER if longest_step(n) is not None and longest_step(n) >= geoms[n]['tt_cap']]
    assert {(geoms[n]['stage_f'], geoms[n]['stage_l']) for n in past} == {(1, 1), (1, 0), (0, 0)}


def test_finish_stage_never_staged_without_front_stage():
    """process_fused_kernel<false, true> does not exist: no shape may ask for it.  obs_dim 1..19 over fixed-horizon and
    variable-length shapes on both sides of the 160 KB shared-memory budget."""
    lib = _library()
    seen = set()
    for Do in range(1, 20):
        shapes = []
        for M in (1, 2, 40, 600, 5000):
            for E in (1, 2, 20, 40, 600):
                for H in (1, 5, 100, 200, 600, 1100, 1500, 4000):
                    shapes.append((M, E, H, Do, E * H, 0))
        for H in range(1, 20000, 37):
            shapes.append((1, 1, H, Do, H, 0))
            shapes.append((40, 20, H, Do, 20 * H, 0))
        for NS in range(4, 40000, 52):
            for M, P in ((1, 1), (2, 30), (3, 15960), (40, 3980)):
                shapes.append((M, min(P, NS), 0, Do, NS, 1))
        for s in shapes:
            g = launch_info(lib, *s)
            assert not (g['stage_f'] == 0 and g['stage_l'] == 1), (s, g)
            seen.add((g['stage_f'], g['stage_l']))
    assert seen == {(1, 1), (1, 0), (0, 0)}


def test_launch_info_validates_arguments():
    lib = _library()
    out = (ctypes.c_int32 * 8)()
    assert lib.promp_process_launch_info(1, 1, 10, 20, 10, 0, out) == -1                 # obs_dim past PS_MAXCOL
    assert lib.promp_process_launch_info(1, 2, 10, 2, 10, 0, out) == -1                  # fixed horizon: NS != E*H
    assert lib.promp_process_launch_info(1, 2, 10, 2, 20, 0, None) == -1
    assert lib.promp_process_launch_info(0, 2, 10, 2, 20, 0, out) == -1


# --------------------------------------------------------------------------------------------------------- oracle
def rel_err(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def oracle_task(paths, discount, gae_lambda, normalize_adv, positive_adv):
    """One task through oracle.numpy_half.SampleProcessor + LinearFeatureBaseline, plus its baseline fitted values and the
    per-task statistics row of promp_process_samples (with a scale row for the summation-order tolerance)."""
    from oracle import numpy_half as nh
    paths = [dict(observations=np.asarray(p['observations'], np.float64), rewards=np.asarray(p['rewards'], np.float64),
                  actions=np.zeros((len(p['rewards']), 1)), env_infos={}, agent_infos={}) for p in paths]
    sp = nh.SampleProcessor(nh.LinearFeatureBaseline(REG), discount, gae_lambda, normalize_adv, positive_adv)
    data, paths = sp.compute_samples_data(paths)
    feats = np.concatenate([nh.baseline_features(p['observations']) for p in paths])
    w = np.asarray(sp.baseline._coeffs)
    R0 = np.array([p['returns'][0] for p in paths])
    G = np.array([p['rewards'].sum() for p in paths])
    r = data['rewards']
    stats = np.array([R0.sum(), G.sum(), (G * G).sum(), G.max(), G.min(), r.sum(), (r * r).sum(), REG])
    scale = np.array([np.abs(R0).sum(), np.abs(G).sum(), (G * G).sum(), np.abs(G).max(), np.abs(G).max(), np.abs(r).sum(),
                      (r * r).sum(), REG])
    return dict(returns=data['returns'], adv=data['advantages'], feats=feats, fitted=feats.dot(w), stats=stats,
                stats_scale=scale, paths=paths)


def compare_task(name, m, got_ret, got_adv, got_coeffs, got_stats, want):
    R = want['returns']
    np.testing.assert_allclose(got_ret, R, rtol=2e-7, atol=1e-6 * np.abs(R).max(), err_msg='%s task %d returns' % (name, m))
    e = rel_err(got_adv, want['adv'])
    assert e < 1e-5, ('%s task %d advantages' % (name, m), e)
    e = rel_err(want['feats'].dot(got_coeffs), want['fitted'])
    assert e < FIT_BAR, ('%s task %d baseline fitted values' % (name, m), e)
    # rtol 1e-9, plus a floor for float64 sums taken in a different order (~n eps sum|x|, n <= 15 000 terms)
    d = np.abs(np.asarray(got_stats[:7]) - want['stats'][:7])
    bar = 1e-9 * np.abs(want['stats'][:7]) + 1e-11 * want['stats_scale'][:7]
    assert np.all(d <= bar), ('%s task %d stats' % (name, m), got_stats, want['stats'])
    assert got_stats[7] == REG, ('%s task %d reg_used' % (name, m), got_stats[7])


# --------------------------------------------------------------------------------------------------------- GPU tests
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _ticket_headers_zero(torch):
    """Every cached processing workspace starts with the per-task arrival tickets; each launch must leave them zero."""
    from promp_b200.samplers.meta_sample_processor import _WS_CACHE
    torch.cuda.synchronize()
    assert _WS_CACHE
    return all(int(torch.count_nonzero(ws[:TICKET_HEADER_DOUBLES])) == 0 for ws in _WS_CACHE.values())


def _origin_seeking_policy(M):
    """theta with mean ~= -100 * obs through the (near-linear) tanh layers and sigma = e^-10: on normalize(MetaPointEnv)
    (a_env = clip(0.01 a, +-0.1)) the point walks 0.1 per step towards the origin and lands within 0.01 of it, so paths
    end early, after <= 21 steps."""
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


class _Case(object):
    """Device state of one case, built once; launch() runs the kernel on it (again) and returns host copies of what it
    wrote; check(out) compares them with the oracle."""

    def __init__(self, torch, name):
        from promp_b200.samplers import MetaSampleProcessor
        from promp_b200.baselines import LinearFeatureBaseline
        self.name, self.phase = name, None
        if name in FIXED:
            M, E, H, Do, disc, lam, norm, pos = FIXED[name]
            self.hyper = (disc, lam, norm, pos)
            self.tasks = host_inputs(name)
            self.paths = OrderedDict((m, [dict(observations=p['observations'], actions=np.zeros((H, 1)), rewards=p['rewards'],
                                               env_infos={}, agent_infos={}) for p in task]) for m, task in enumerate(self.tasks))
        elif name == 'ragged_ws64':
            self._build_ragged(torch)
        elif name == 'early_term':
            self._build_early_term()
        elif name != 'baseline_fit':
            raise KeyError(name)
        if name != 'baseline_fit':
            self.proc = MetaSampleProcessor(LinearFeatureBaseline(REG), *self.hyper)

    def _build_ragged(self, torch):
        from promp_b200.samplers.device_data import RaggedPhaseData
        self.hyper = RAGGED_HYPER
        self.tasks = host_inputs('ragged_ws64')
        ph = RaggedPhaseData([[len(p['rewards']) for p in t] for t in self.tasks], 2, 1, torch.device('cuda'))
        M, N = ph.M, ph.N
        self.obs_in = np.full((M, N, 2), 1e3, np.float32)           # padding rows poisoned: they must not contribute
        self.rew_in = np.full((M, N), 1e4, np.float32)
        for m, t in enumerate(self.tasks):
            n = int(ph.n_valid_host[m])
            self.obs_in[m, :n] = np.concatenate([p['observations'] for p in t])
            self.rew_in[m, :n] = np.concatenate([p['rewards'] for p in t])
        ph.obs.copy_(torch.from_numpy(self.obs_in))
        ph.rew.copy_(torch.from_numpy(self.rew_in))
        f32 = dict(dtype=torch.float32, device='cuda')
        ph.returns, ph.adv = torch.full((M, N), 777.0, **f32), torch.full((M, N), 777.0, **f32)
        ph.coeffs = torch.zeros(M, 2 * 2 + 4, dtype=torch.float64, device='cuda')
        ph.stats = torch.zeros(M, 8, dtype=torch.float64, device='cuda')
        self.phase = ph

    def _build_early_term(self):
        from promp_b200.envs import normalize, MetaPointEnv
        from promp_b200.samplers import MetaSampler
        M, E, H = EARLY_TERM['M'], EARLY_TERM['E'], EARLY_TERM['H']
        self.hyper = (0.99, 1.0, True, False)
        policy = _origin_seeking_policy(M)
        sampler = MetaSampler(env=normalize(MetaPointEnv()), policy=policy, rollouts_per_meta_task=E, meta_batch_size=M,
                              max_path_length=H, reset_mode='device', seed=5)
        assert sampler._fused_early_ok()
        sampler.update_tasks()
        policy.switch_to_pre_update()
        self.paths = sampler.obtain_samples()
        # the lazy host path list the sampler hands to reference-style callers, copied before any processing
        self.tasks = [[dict(observations=np.array(p['observations'], np.float64), rewards=np.array(p['rewards'], np.float64))
                       for p in self.paths[m]] for m in range(M)]
        assert max(len(p['rewards']) for t in self.tasks for p in t) <= 21

    def launch(self):
        from promp_b200.samplers.meta_sample_processor import run_process_kernel
        if self.name == 'baseline_fit':
            from promp_b200.baselines import LinearFeatureBaseline
            paths = host_inputs(self.name)[0]
            base = LinearFeatureBaseline(REG)
            base.fit([dict(observations=p['observations'], returns=p['returns']) for p in paths])
            coeffs = np.asarray(base.get_param_values(), dtype=np.float64).copy()
            return dict(coeffs=coeffs, pred=np.concatenate([base.predict(p) for p in paths]))
        if self.name == 'ragged_ws64':
            run_process_kernel(self.phase, self.hyper[0], self.hyper[1], REG, 1, self.hyper[2], self.hyper[3])
        elif self.phase is None:
            # host paths (fixed horizon) or the sampler's device phase (early_term); later launches re-process that phase
            self.phase = self.proc.process_samples(self.paths)[0].phase
        else:
            self.proc.process_phase(self.phase)
        ph = self.phase
        return dict(returns=ph.returns.cpu().numpy(), adv=ph.adv.cpu().numpy(), coeffs=ph.coeffs.cpu().numpy(),
                    stats=ph.stats.cpu().numpy(), log_terms=self.proc.device_log_terms(ph).cpu().numpy())

    # ---- oracle comparison
    def check(self, out):
        from oracle import numpy_half as nh
        if self.name == 'baseline_fit':
            paths = host_inputs(self.name)[0]
            ref = nh.LinearFeatureBaseline(REG)
            ref.fit(paths)
            feats = np.concatenate([nh.baseline_features(p['observations']) for p in paths])
            want = np.concatenate([ref.predict(p) for p in paths])
            e = rel_err(feats.dot(out['coeffs']), want)
            assert e < FIT_BAR, ('fitted values', e)
            e = rel_err(out['pred'], feats.dot(out['coeffs']))       # promp_baseline_predict evaluates Phi w
            assert e < 1e-12, ('predict', e)
            return
        ph = self.phase
        all_paths = []
        for m, task in enumerate(self.tasks):
            want = oracle_task(task, *self.hyper)
            n = len(want['returns'])
            compare_task(self.name, m, out['returns'][m, :n], out['adv'][m, :n], out['coeffs'][m], out['stats'][m], want)
            all_paths += want['paths']
            if self.name == 'ragged_ws64':
                assert np.all(out['adv'][m, n:] == 0.0), 'advantages of padding rows must be 0'
                assert np.all(out['returns'][m, n:] == 777.0), 'returns past n_valid must stay untouched'
        if self.name == 'ragged_ws64':
            np.testing.assert_array_equal(ph.obs.cpu().numpy(), self.obs_in)
            np.testing.assert_array_equal(ph.rew.cpu().numpy(), self.rew_in)
        # the logged path statistics (samplers/base.py:135-149) from the per-task rows
        ps = nh.path_stats(all_paths)
        want = [ps[k] for k in ('AverageDiscountedReturn', 'AverageReturn', 'NumTrajs', 'StdReturn', 'MaxReturn', 'MinReturn')]
        np.testing.assert_allclose(out['log_terms'], want, rtol=1e-9, atol=1e-12, err_msg=self.name + ' path statistics')


@pytest.fixture(scope='module')
def forward_pass():
    """Every case once, in CASE_ORDER, on the processor's shared cached workspace."""
    torch = _cuda()
    torch.cuda.set_device(0)
    done = OrderedDict()
    for name in CASE_ORDER:
        case = _Case(torch, name)
        out = case.launch()
        done[name] = (case, out, _ticket_headers_zero(torch))
    return done


@pytest.mark.gpu
@pytest.mark.parametrize('name', CASE_ORDER)
def test_process_case_matches_oracle(forward_pass, name):
    from promp_b200 import _lib
    lib = _lib.load()
    check_geometry(lib, name)
    case, out, headers_zero = forward_pass[name]
    if case.phase is not None:            # the launch really had the shape the geometry pin names
        ph = case.phase
        got = launch_info(lib, ph.M, ph.E, 0 if ph.H is None else ph.H, ph.obs_dim, ph.N, ph.H is None)
        assert got == launch_info(lib, *case_shape(name)), (name, got)
    assert headers_zero, name + ': ticket header not left zero'
    case.check(out)


@pytest.mark.gpu
def test_shared_workspace_reuse_in_reverse_order(forward_pass):
    """The cases again, in reverse order, on the same cached workspace the forward pass left behind: every output is
    bit-identical to the first pass and the ticket header reads zero after every launch."""
    torch = _cuda()
    for name in reversed(CASE_ORDER):
        case, first, _ = forward_pass[name]
        again = case.launch()
        assert _ticket_headers_zero(torch), name + ': ticket header not left zero'
        assert set(again) == set(first)
        for k in first:
            a, b = np.ascontiguousarray(first[k]), np.ascontiguousarray(again[k])
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (name, k)
