"""NormalizedEnv / normalize (ref: meta_policy_search/envs/normalized_env.py:6-126).

On the device the wrapper is the affine action map + clip that the env kernels always apply
(csrc/envs.cuh: normalized_action); observation / reward running normalisation (off by default in
the reference, :23-24) is out of scope and rejected loudly.
"""
import numpy as np

from promp_b200.envs.base import Box


class NormalizedEnv(object):
    def __init__(self, env, scale_reward=1., normalize_obs=False, normalize_reward=False, obs_alpha=0.001,
                 reward_alpha=0.001, normalization_scale=10.):
        if normalize_obs or normalize_reward:
            raise NotImplementedError("promp_b200: running obs/reward normalisation is out of scope (reference default is off)")
        if float(normalization_scale) != 10.0:
            raise NotImplementedError("promp_b200: the device env kernels implement normalization_scale=10 only")
        if not hasattr(env, 'device_spec'):
            raise TypeError("promp_b200.normalize needs a device env (promp_b200.envs.*, or your own dynamics as a "
                            "promp_b200.envs.CudaMetaEnv); got %r" % (env,))
        self._wrapped_env = env
        self._normalization_scale = normalization_scale
        self._scale_reward = 1

    @property
    def action_space(self):
        ub = np.ones(self._wrapped_env.action_space.shape) * self._normalization_scale
        return Box(-1 * ub, ub, dtype=np.float32)

    def __getattr__(self, attr):
        if attr.startswith('__') or attr == '_wrapped_env':
            raise AttributeError(attr)
        return getattr(self._wrapped_env, attr)

    def device_spec(self):
        spec = dict(self._wrapped_env.device_spec())
        spec['normalized'] = True
        return spec

    def __getstate__(self):
        return dict(env=self._wrapped_env)

    def __setstate__(self, d):
        self.__init__(d['env'])


normalize = NormalizedEnv
