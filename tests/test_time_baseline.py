"""Every baseline the reference accepts, on the GPU:

  - LinearTimeBaseline (baselines/linear_baseline.py:109-126) as the processing kernel's LINEAR_TIME kind, against the
    float64 oracle (oracle/time_baseline.py, pinned to the reference by test_time_baseline_oracle.py) on every launch
    geometry case of test_process_geometry.py, with that file's bars;
  - the reference's own LinearTimeBaseline tests (tests/test_baselines.py:112-150) on the device class;
  - any other baseline object (samplers/base.py:99-108 asks only for fit / predict): fitted and evaluated on the host in
    the reference's call order, everything else on the device (the GIVEN kind);
  - Trainer.train() with either: the time baseline replays as a CUDA graph, a host baseline trains eagerly.
"""
import pickle

import numpy as np
import pytest

import test_process_geometry as pg

REG = pg.REG


def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


# ------------------------------------------------------------------------------------- 1. time kind vs the oracle
def oracle_task_time(paths, discount, gae_lambda, normalize_adv, positive_adv):
    """pg.oracle_task with LinearTimeBaseline: returns and statistics do not depend on the baseline, the advantages and
    the fitted values Phi w come from the time oracle."""
    from oracle import numpy_half as nh
    from oracle.time_baseline import LinearTimeBaseline, time_features
    want = pg.oracle_task(paths, discount, gae_lambda, normalize_adv, positive_adv)
    paths = [dict(observations=np.asarray(p['observations'], np.float64), rewards=np.asarray(p['rewards'], np.float64),
                  actions=np.zeros((len(p['rewards']), 1)), env_infos={}, agent_infos={}) for p in paths]
    sp = nh.SampleProcessor(LinearTimeBaseline(REG), discount, gae_lambda, normalize_adv, positive_adv)
    data, paths = sp.compute_samples_data(paths)
    feats = np.concatenate([time_features(len(p['rewards'])) for p in paths])
    want.update(adv=data['advantages'], feats=feats, fitted=feats.dot(np.asarray(sp.baseline._coeffs)))
    return want


def _time_case(torch, name):
    """Run one geometry case of test_process_geometry.py with the time kind; returns (case, host outputs)."""
    from promp_b200.baselines import LinearTimeBaseline
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    case = pg._Case(torch, name)
    if name == 'baseline_fit':
        paths = pg.host_inputs(name)[0]
        base = LinearTimeBaseline(REG)
        base.fit([dict(observations=p['observations'], returns=p['returns']) for p in paths])
        return case, dict(coeffs=np.asarray(base.get_param_values(), np.float64).copy(),
                          pred=np.concatenate([base.predict(p) for p in paths]))
    case.proc = MetaSampleProcessor(LinearTimeBaseline(REG), *case.hyper)
    if name == 'ragged_ws64':
        run_process_kernel(case.phase, case.hyper[0], case.hyper[1], REG, 2, case.hyper[2], case.hyper[3])
    else:
        case.phase = case.proc.process_samples(case.paths)[0].phase
        assert case.proc.baseline.get_param_values() is not None
    ph = case.phase
    assert tuple(ph.coeffs.shape) == (ph.M, 4)
    return case, dict(returns=ph.returns.cpu().numpy(), adv=ph.adv.cpu().numpy(), coeffs=ph.coeffs.cpu().numpy(),
                      stats=ph.stats.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize('name', pg.CASE_ORDER)
def test_time_kind_matches_oracle(name):
    from oracle.time_baseline import LinearTimeBaseline, time_features
    torch = _cuda()
    case, out = _time_case(torch, name)
    assert pg._ticket_headers_zero(torch), name + ': ticket header not left zero'
    if name == 'baseline_fit':
        paths = pg.host_inputs(name)[0]
        ref = LinearTimeBaseline(REG)
        ref.fit(paths)
        feats = np.concatenate([time_features(len(p['rewards'])) for p in paths])
        want = np.concatenate([ref.predict(p) for p in paths])
        assert pg.rel_err(feats.dot(out['coeffs']), want) < pg.FIT_BAR
        assert pg.rel_err(out['pred'], feats.dot(out['coeffs'])) < 1e-12       # promp_baseline_predict_ex evaluates Phi w
        return
    for m, task in enumerate(case.tasks):
        want = oracle_task_time(task, *case.hyper)
        n = len(want['returns'])
        pg.compare_task(name, m, out['returns'][m, :n], out['adv'][m, :n], out['coeffs'][m], out['stats'][m], want)
        if case.phase.H is None:
            assert np.all(out['adv'][m, n:] == 0.0), 'advantages of padding rows must be 0'
    # the baseline object holds the last task's coefficients (a lazy view of the device buffer)
    if name != 'ragged_ws64':
        np.testing.assert_array_equal(np.asarray(case.proc.baseline.get_param_values()), out['coeffs'][-1])


# ------------------------------------------------------------------- 2. the reference's LinearTimeBaseline tests
def _reference_tasks(seed):
    """tests/test_baselines.py:113-117 (seeded)."""
    rng = np.random.RandomState(seed)
    base_path = np.arange(-4.0, 22.0, step=.6)
    task1 = [{'discounted_rewards': base_path + rng.normal(scale=2, size=base_path.shape), 'observations': base_path}
             for _ in range(10)]
    task2 = [{'discounted_rewards': base_path ** 3 + rng.normal(scale=2, size=base_path.shape), 'observations': base_path}
             for _ in range(10)]
    return [task1, task2]


def _sq_error(baseline, task):
    return sum(np.sum(np.square(baseline.predict(p) - p['discounted_rewards'])) for p in task)


@pytest.mark.gpu
def test_reference_testFit():
    """tests/test_baselines.py:112-129, plus the fit against the oracle and zeros before the first fit."""
    from promp_b200.baselines import LinearTimeBaseline
    from oracle.time_baseline import LinearTimeBaseline as OracleTime
    _cuda()
    linear = LinearTimeBaseline()
    for task in _reference_tasks(0):
        unfit_error = np.sum([np.sum(p['discounted_rewards'] ** 2) for p in task])
        linear.fit(task, target_key='discounted_rewards')
        fit_error = _sq_error(linear, task)
        assert 2 * fit_error < unfit_error
        ref = OracleTime()
        ref.fit(task, target_key='discounted_rewards')
        got = np.concatenate([linear.predict(p) for p in task])
        want = np.concatenate([ref.predict(p) for p in task])
        assert pg.rel_err(got, want) < pg.FIT_BAR
    fresh = LinearTimeBaseline()
    pred = fresh.predict(_reference_tasks(1)[0][0])
    assert pred.shape == (44,) and np.all(pred == 0.0)


@pytest.mark.gpu
def test_reference_testSerialize():
    """tests/test_baselines.py:131-150."""
    from promp_b200.baselines import LinearTimeBaseline
    _cuda()
    linear = LinearTimeBaseline()
    for task in _reference_tasks(2):
        linear.fit(task, target_key='discounted_rewards')
        fit_error_pre = _sq_error(linear, task)
        linear = pickle.loads(pickle.dumps(linear))
        fit_error_post = _sq_error(linear, task)
        assert fit_error_pre == fit_error_post


# ----------------------------------------------------------------------------------------- 3. host baselines
class NumpyFeatureBaseline(object):
    """LinearFeatureBaseline's semantics in plain numpy (no device_kind): MetaSampleProcessor must run it on the host."""

    def __init__(self, reg_coeff=REG):
        from oracle import numpy_half as nh
        self._impl = nh.LinearFeatureBaseline(reg_coeff)

    def fit(self, paths, target_key='returns'):
        self._impl.fit(paths, target_key=target_key)

    def predict(self, path):
        return self._impl.predict(path)

    def log_diagnostics(self, paths, prefix=''):
        pass


class RecordingBaseline(object):
    """Records every call; predicts zeros."""

    def __init__(self):
        self.calls = []

    def fit(self, paths, target_key='returns'):
        self.calls.append(('fit', target_key, [(np.array(p['rewards']), np.array(p['returns'])) for p in paths]))

    def predict(self, path):
        self.calls.append(('predict', np.array(path['rewards'])))
        return np.zeros(len(path['observations']))


class KnownBaseline(object):
    """Predicts a fixed function of the path (float64); fit does nothing."""

    def fit(self, paths, target_key='returns'):
        pass

    def predict(self, path):
        r = np.asarray(path['rewards'], np.float64)
        return 0.9 * np.cumsum(r[::-1])[::-1] + 0.01 * len(r) - 0.003 * np.arange(len(r))


def _host_paths(layout):
    """Seeded host paths: fixed (3 tasks x 20 paths x 100 steps, obs_dim 4) or ragged (variable lengths, obs_dim 3)."""
    rng = np.random.RandomState(5 if layout == 'fixed' else 6)
    if layout == 'fixed':
        lens, Do = [[100] * 20] * 3, 4
    else:
        lens, Do = [[5, 17, 1, 30, 12, 200], [40, 3], [9, 9, 9, 25, 2, 2, 31, 140]], 3
    out = {}
    for m, task in enumerate(lens):
        out[m] = [dict(observations=pg._walk(rng, L, Do), actions=np.zeros((L, 1)), rewards=pg._rewards(rng, L),
                       env_infos={}, agent_infos={}) for L in task]
    return out


def _phase(torch, layout):
    from promp_b200.samplers.meta_sample_processor import _phase_from_host_paths
    return _phase_from_host_paths(_host_paths(layout), torch.device('cuda'))


def _task_bounds(phase, m):
    if phase.H is None:
        return phase.path_off_host[m][:int(phase.n_paths_host[m]) + 1]
    return np.arange(phase.E + 1) * phase.H


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['fixed', 'ragged'])
@pytest.mark.parametrize('normalize_adv,positive_adv', [(False, False), (True, False), (True, True), (False, True)])
def test_numpy_feature_baseline_matches_device(layout, normalize_adv, positive_adv):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.samplers import MetaSampleProcessor
    torch = _cuda()
    phase = _phase(torch, layout)
    MetaSampleProcessor(LinearFeatureBaseline(REG), 0.99, 0.97, normalize_adv, positive_adv).process_phase(phase)
    want = {k: getattr(phase, k).cpu().numpy().copy() for k in ('returns', 'adv', 'stats')}
    host = NumpyFeatureBaseline()
    MetaSampleProcessor(host, 0.99, 0.97, normalize_adv, positive_adv).process_phase(phase)
    got = {k: getattr(phase, k).cpu().numpy() for k in ('returns', 'adv', 'stats')}
    np.testing.assert_array_equal(got['returns'], want['returns'])
    for m in range(phase.M):
        n = int(_task_bounds(phase, m)[-1])
        assert pg.rel_err(got['adv'][m, :n], want['adv'][m, :n]) < 1e-4, (layout, m)
        np.testing.assert_allclose(got['stats'][m, :7], want['stats'][m, :7], rtol=1e-4, atol=1e-4)
        assert got['stats'][m, 7] == 0.0
        if layout == 'ragged':
            assert np.all(got['adv'][m, n:] == 0.0)
    assert host._impl._coeffs is not None        # left fitted on the last task, as in the reference


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['fixed', 'ragged'])
def test_host_baseline_call_order(layout):
    """M fits in task order, each on that task's paths with the device returns, then one predict per path in order."""
    from promp_b200.samplers import MetaSampleProcessor
    torch = _cuda()
    phase = _phase(torch, layout)
    rec = RecordingBaseline()
    MetaSampleProcessor(rec, 0.99, 1.0, True, False).process_phase(phase)
    rew, ret = phase.rew.cpu().numpy(), phase.returns.cpu().numpy()
    want = []
    for m in range(phase.M):
        b = _task_bounds(phase, m)
        segs = [slice(int(b[k]), int(b[k + 1])) for k in range(len(b) - 1)]
        want.append(('fit', segs, m))
        want += [('predict', s, m) for s in segs]
    assert [c[0] for c in rec.calls] == [w[0] for w in want]
    for call, (kind, segs, m) in zip(rec.calls, want):
        if kind == 'fit':
            assert call[1] == 'returns' and len(call[2]) == len(segs)
            for (r, R), s in zip(call[2], segs):
                np.testing.assert_array_equal(r, rew[m, s])
                np.testing.assert_array_equal(R, ret[m, s])
        else:
            np.testing.assert_array_equal(call[1], rew[m, segs])


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['fixed', 'ragged'])
@pytest.mark.parametrize('normalize_adv,positive_adv', [(False, False), (True, True)])
def test_host_baseline_values_give_oracle_gae(layout, normalize_adv, positive_adv):
    from oracle import numpy_half as nh
    from promp_b200.samplers import MetaSampleProcessor
    torch = _cuda()
    phase = _phase(torch, layout)
    MetaSampleProcessor(KnownBaseline(), 0.98, 0.95, normalize_adv, positive_adv).process_phase(phase)
    adv = phase.adv.cpu().numpy()
    sp = nh.SampleProcessor(KnownBaseline(), 0.98, 0.95, normalize_adv, positive_adv)
    for m, task in _host_paths(layout).items():
        data, _ = sp.compute_samples_data([dict(p) for p in task])
        n = len(data['advantages'])
        assert pg.rel_err(adv[m, :n], data['advantages']) < 1e-5, (layout, m)


# --------------------------------------------------------------------------------------------- 4. the Trainer
def _trainer(torch, baseline, graph, seed=3, M=4, E=3, H=30):
    from promp_b200.envs import normalize, MetaPointEnvCorner
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    np.random.seed(seed)
    torch.manual_seed(seed)
    env = normalize(MetaPointEnvCorner())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=baseline, discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3,
                 num_ppo_steps=5, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    return Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=3,
                   num_inner_grad_steps=1, use_cuda_graph=graph)


def _train(torch, tr, tmp_path):
    from promp_b200.utils import logger
    th0 = tr.policy.theta.clone()
    try:
        logger.configure(dir=str(tmp_path), format_strs=['json'], snapshot_mode='none')
        tr.train()
        kv = dict(logger.last_dump())
    finally:
        logger.reset()
    assert torch.isfinite(tr.policy.theta).all() and not torch.equal(tr.policy.theta, th0)
    for k in ('LossBefore', 'LossAfter', 'Step_0-AverageReturn', 'Step_1-AverageReturn'):
        assert np.isfinite(kv[k]), k
    return kv


@pytest.mark.gpu
def test_trainer_replays_time_baseline_as_graph(tmp_path):
    from promp_b200.baselines import LinearTimeBaseline
    torch = _cuda()
    runs = []
    for i in range(2):
        tr = _trainer(torch, LinearTimeBaseline(), 'auto')
        assert tr.graph_capturable()
        kv = _train(torch, tr, tmp_path / str(i))
        assert tr._graph_step is not None
        assert np.asarray(tr.baseline.get_param_values()).shape == (4,)
        runs.append((tr.policy.theta.clone(), kv))
    assert torch.equal(runs[0][0], runs[1][0])
    for k, v in runs[0][1].items():
        if 'Time' not in k and isinstance(v, (float, int, np.floating)):
            assert v == runs[1][1][k] or (np.isnan(v) and np.isnan(runs[1][1][k])), k


@pytest.mark.gpu
def test_trainer_with_host_baseline_runs_eagerly(tmp_path):
    torch = _cuda()
    tr = _trainer(torch, NumpyFeatureBaseline(), 'auto')
    assert not tr.graph_capturable()
    _train(torch, tr, tmp_path / 'eager')
    assert tr._graph_step is None and tr.baseline._impl._coeffs is not None
    tr = _trainer(torch, NumpyFeatureBaseline(), True)
    with pytest.raises(ValueError, match='device baseline'):
        tr.train()
