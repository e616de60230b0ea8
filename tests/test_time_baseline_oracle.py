"""LinearTimeBaseline (baselines/linear_baseline.py:109-126) without a GPU: the float64 oracle (oracle/time_baseline.py)
against the unmodified reference's outputs (tests/golden/time_baseline.npz, written by
oracle/make_time_baseline_golden.py), and the host-side behaviour of promp_b200.baselines.LinearTimeBaseline."""
import os
import pickle

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'time_baseline.npz')
CASES = ('fixed', 'fixed_gae', 'variable', 'length_one')


def golden_tasks(g, name):
    """Per task: list of {observations, rewards} paths rebuilt from the fixture (the time baseline reads only the path
    lengths of the observations)."""
    pre = 'case_%s_' % name
    lens, rew = g[pre + 'path_len'], g[pre + 'rew'].astype(np.float64)
    tasks, k, n = [], 0, 0
    for P in g[pre + 'n_paths']:
        task = []
        for L in lens[k:k + P]:
            task.append(dict(observations=np.zeros((int(L), 2)), actions=np.zeros((int(L), 1)), rewards=rew[n:n + L],
                             env_infos={}, agent_infos={}))
            n += int(L)
        k += P
        tasks.append(task)
    return tasks


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_golden(name):
    from oracle import numpy_half as nh
    from oracle.time_baseline import LinearTimeBaseline
    g = np.load(GOLDEN)
    pre = 'case_%s_' % name
    cfg = [g[pre + 'cfg_' + k].item() for k in ('discount', 'gae_lambda', 'normalize_adv', 'positive_adv')]
    sp = nh.SampleProcessor(LinearTimeBaseline(), *cfg)
    coeffs, returns, adv = [], [], []
    for task in golden_tasks(g, name):
        data, _ = sp.compute_samples_data(task)
        coeffs.append(np.array(sp.baseline._coeffs))
        returns.append(data['returns'])
        adv.append(data['advantages'])
    want_c = g[pre + 'coeffs']
    np.testing.assert_allclose(np.stack(coeffs), want_c, rtol=1e-9, atol=1e-9 * np.abs(want_c).max(), err_msg=name)
    np.testing.assert_allclose(np.concatenate(returns), g[pre + 'returns'], rtol=1e-12, atol=1e-12, err_msg=name)
    want_a = g[pre + 'advantages']
    np.testing.assert_allclose(np.concatenate(adv), want_a, rtol=1e-6, atol=1e-6 * np.abs(want_a).max(), err_msg=name)


def test_length_one_paths_fit_only_the_constant():
    """All paths of one step: t = 0 everywhere, so the reference's ridge solve leaves the three time coefficients at 0."""
    g = np.load(GOLDEN)
    c = g['case_length_one_coeffs']
    assert np.all(c[:, :3] == 0.0) and np.all(c[:, 3] != 0.0)


def test_device_class_host_side():
    """The parts of promp_b200.baselines.LinearTimeBaseline that never launch a kernel: kind, features, zeros before the
    first fit (linear_baseline.py:31-33), parameters, pickling."""
    from promp_b200.baselines import LinearTimeBaseline, LinearFeatureBaseline
    from oracle.time_baseline import time_features
    b = LinearTimeBaseline(reg_coeff=1e-4)
    assert b.device_kind == 2 and LinearFeatureBaseline.device_kind == 1
    path = dict(observations=np.arange(44.0), rewards=np.ones(44))
    np.testing.assert_array_equal(b._features(path), time_features(44))
    pred = b.predict(path)
    assert pred.shape == (44,) and np.all(pred == 0.0)
    assert b.get_param_values() is None
    b.set_params(np.array([1.0, 2.0, 3.0, 4.0]))
    c = pickle.loads(pickle.dumps(b))
    assert c._reg_coeff == 1e-4 and np.array_equal(c.get_param_values(), [1.0, 2.0, 3.0, 4.0])
    c.log_diagnostics([path])
