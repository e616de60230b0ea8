"""CPU restatement of the reference's LinearTimeBaseline.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

ref: baselines/linear_baseline.py:6-80 (LinearBaseline: fit / predict) and :109-126 (LinearTimeBaseline._features).  It
plugs into oracle.numpy_half.SampleProcessor like numpy_half.LinearFeatureBaseline.  Pinned against the unmodified
reference by tests/test_time_baseline_oracle.py (fixture written by oracle/make_time_baseline_golden.py).
"""
import numpy as np


def time_features(n):
    """ref: baselines/linear_baseline.py:122-126 for a path of n steps: [t, t^2, t^3, 1], t = step / 100."""
    t = np.arange(n).reshape(-1, 1) / 100.0
    return np.concatenate([t, t ** 2, t ** 3, np.ones((n, 1))], axis=1)


class LinearTimeBaseline(object):
    """ref: baselines/linear_baseline.py:109-126 with the fit / predict of :17-77."""

    def __init__(self, reg_coeff=1e-5):
        self._coeffs = None
        self._reg_coeff = reg_coeff

    def fit(self, paths, target_key='returns'):            # ref :55-77
        featmat = np.concatenate([time_features(len(p["observations"])) for p in paths], axis=0)
        target = np.concatenate([p[target_key] for p in paths], axis=0)
        reg = self._reg_coeff
        for _ in range(5):
            self._coeffs = np.linalg.lstsq(featmat.T.dot(featmat) + reg * np.identity(featmat.shape[1]),
                                           featmat.T.dot(target), rcond=-1)[0]
            if not np.any(np.isnan(self._coeffs)):
                break
            reg *= 10

    def predict(self, path):                               # ref :17-33
        if self._coeffs is None:
            return np.zeros(len(path["observations"]))
        return time_features(len(path["observations"])).dot(self._coeffs)
