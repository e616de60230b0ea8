"""LinearFeatureBaseline and LinearTimeBaseline (ref: meta_policy_search/baselines/linear_baseline.py:6-126).

On the hot path the fit (float64 Gram + Cholesky with the reference's ridge / NaN-retry rule) and the
prediction happen inside promp_process_samples, one fit per task, for the kind the class names (`device_kind`); this
object carries `reg_coeff` in, and receives the coefficients of the LAST fitted task out - exactly the state the
reference's shared baseline object is left in after MetaSampleProcessor.process_samples
(samplers/meta_sample_processor.py:31-34).  Called on its own (the reference's tests/test_baselines.py:67-150 do),
`fit(paths, target_key)` and `predict(path)` run the same float64 Gram / ridge-solve / feature code through the
standalone entry points promp_baseline_fit_ex / promp_baseline_predict_ex; `_features` is a host helper for diagnostics.
"""
import numpy as np


class LinearBaseline(object):
    """linear_baseline.py:6-80: what both linear baselines share.  Subclasses set `device_kind` and `_features`."""
    device_kind = None

    def __init__(self, reg_coeff=1e-5):
        self._coeffs = None
        self._reg_coeff = reg_coeff

    def get_param_values(self, **tags):
        return self._coeffs

    def set_params(self, value, **tags):
        self._coeffs = value

    def predict(self, path):
        """linear_baseline.py:17-33: zeros if never fitted, else features . coeffs (on the device)."""
        if self._coeffs is None:
            return np.zeros(len(path["observations"]))
        from promp_b200.samplers.meta_sample_processor import predict_baseline_on_path
        return predict_baseline_on_path(path, np.asarray(self._coeffs, dtype=np.float64), self.device_kind)

    def fit(self, paths, target_key='returns'):
        """linear_baseline.py:55-77 on a flat list of (variable-length) paths, through promp_baseline_fit_ex."""
        from promp_b200.samplers.meta_sample_processor import fit_baseline_on_paths
        self._coeffs = fit_baseline_on_paths(paths, target_key, self._reg_coeff, self.device_kind)

    def log_diagnostics(self, paths, prefix=''):
        pass

    def __getstate__(self):
        coeffs = None if self._coeffs is None else np.asarray(self._coeffs, dtype=np.float64)   # a lazy device view -> numbers
        return dict(reg_coeff=self._reg_coeff, coeffs=coeffs)

    def __setstate__(self, d):
        self._reg_coeff, self._coeffs = d['reg_coeff'], d['coeffs']


class LinearFeatureBaseline(LinearBaseline):
    """Features [clip(o), clip(o)^2, t, t^2, t^3, 1], t = step / 100 (linear_baseline.py:83-106); coefficients 2*Do+4."""
    device_kind = 1

    def _features(self, path):
        obs = np.clip(path["observations"], -10, 10)
        n = len(path["observations"])
        t = np.arange(n).reshape(-1, 1) / 100.0
        return np.concatenate([obs, obs ** 2, t, t ** 2, t ** 3, np.ones((n, 1))], axis=1)


class LinearTimeBaseline(LinearBaseline):
    """Features [t, t^2, t^3, 1], t = step / 100 restarting in every path (linear_baseline.py:109-126); coefficients [4].
    The observations are never read, only their count per path."""
    device_kind = 2

    def _features(self, path):
        n = len(path["observations"])
        t = np.arange(n).reshape(-1, 1) / 100.0
        return np.concatenate([t, t ** 2, t ** 3, np.ones((n, 1))], axis=1)
