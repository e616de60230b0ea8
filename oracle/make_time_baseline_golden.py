"""Generate tests/golden/time_baseline.npz by running the UNMODIFIED reference LinearTimeBaseline through the reference's
sample processing (SampleProcessor._compute_samples_data, samplers/base.py:99-133, per task as
MetaSampleProcessor.process_samples calls it, samplers/meta_sample_processor.py:31-34).

Like oracle/make_golden.py this imports the reference modules from where they lie (PROMP_REFERENCE_DIR, by default
../reference next to this repository) with the stub packages of oracle/stubs standing in for gym / pyprind /
rand_param_envs.  Nothing from the reference is copied: only its numeric outputs are stored.

Cases: fixed-length paths, variable-length paths, and tasks whose paths all have one step (every time feature but the
constant is 0: the Gram matrix has rank 1 and only the ridge makes the system solvable).

    python oracle/make_time_baseline_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get('PROMP_REFERENCE_DIR', os.path.join(os.path.dirname(ROOT), 'reference'))
OUT = os.path.join(ROOT, 'tests', 'golden', 'time_baseline.npz')

# name -> (per-task path lengths, discount, gae_lambda, normalize_adv, positive_adv)
CASES = {
    'fixed': ([[100] * 5, [100] * 5, [100] * 5], 0.99, 1.0, True, False),
    'fixed_gae': ([[200] * 4, [200] * 4], 0.95, 0.9, False, False),
    'variable': ([[5, 17, 1, 30, 12], [40, 3], [9, 9, 9, 25, 2, 2, 31], [150, 1, 260]], 0.99, 0.97, True, True),
    'length_one': ([[1] * 6, [1] * 3], 0.99, 1.0, False, False),
}
OBS_DIM = 2


def case_paths(name):
    """Seeded float32-representable paths of a case: list (tasks) of lists of {observations, actions, rewards, ...}."""
    lens = CASES[name][0]
    rng = np.random.RandomState(sum(map(ord, name)))
    tasks = []
    for task_lens in lens:
        paths = []
        for L in task_lens:
            obs = np.cumsum(0.3 * rng.randn(L, OBS_DIM), axis=0).astype(np.float32).astype(np.float64)
            rew = (rng.randn(L) * (rng.rand(L) < 0.6) + 0.02 * np.arange(L)).astype(np.float32).astype(np.float64)
            paths.append(dict(observations=obs, actions=np.zeros((L, 1)), rewards=rew, env_infos={}, agent_infos={}))
        tasks.append(paths)
    return tasks


def main():
    if not os.path.isdir(REF):
        raise SystemExit("reference tree %s not present (set PROMP_REFERENCE_DIR)" % REF)
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'stubs'))
    sys.path.insert(0, REF)
    from meta_policy_search.baselines.linear_baseline import LinearTimeBaseline
    from meta_policy_search.samplers.meta_sample_processor import MetaSampleProcessor
    out = {}
    for name, (lens, discount, gae_lambda, normalize_adv, positive_adv) in CASES.items():
        proc = MetaSampleProcessor(baseline=LinearTimeBaseline(), discount=discount, gae_lambda=gae_lambda,
                                   normalize_adv=normalize_adv, positive_adv=positive_adv)
        pre = 'case_%s_' % name
        coeffs, returns, adv, rew = [], [], [], []
        for paths in case_paths(name):
            data, _ = proc._compute_samples_data(paths)
            coeffs.append(np.array(proc.baseline._coeffs, dtype=np.float64))
            returns.append(data['returns'])
            adv.append(data['advantages'])
            rew.append(data['rewards'])
        for k, v in (('discount', discount), ('gae_lambda', gae_lambda), ('normalize_adv', normalize_adv),
                     ('positive_adv', positive_adv)):
            out[pre + 'cfg_' + k] = np.asarray(v)
        out[pre + 'n_paths'] = np.asarray([len(l) for l in lens], dtype=np.int32)
        out[pre + 'path_len'] = np.concatenate([np.asarray(l, dtype=np.int32) for l in lens])
        out[pre + 'rew'] = np.concatenate(rew).astype(np.float32)
        out[pre + 'coeffs'] = np.stack(coeffs)
        out[pre + 'returns'] = np.concatenate(returns)
        out[pre + 'advantages'] = np.concatenate(adv)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays)" % (OUT, len(out)))


if __name__ == '__main__':
    main()
