"""MetaGaussianMLPPolicy with device-resident parameters.

Mirrors the reference's policy container (meta_policy_search/policies/meta_gaussian_mlp_policy.py:9-157,
policies/gaussian_mlp_policy.py:31-184, policies/base.py:164-286): a pre-update parameter set theta
(the tf.Variables) and M post-update parameter sets theta_i' (the placeholders fed by
update_task_parameters).  Both live in HBM as flat float32 vectors in the reference's variable order;
the sampler and the algorithms hand their device pointers straight to the kernels.
"""
import math
from collections import OrderedDict

import numpy as np

from promp_b200 import _lib
from promp_b200.policies.distributions import DiagonalGaussian
from promp_b200.utils import logger

PARAM_NAMES = ('mean_network/hidden_0/kernel', 'mean_network/hidden_0/bias',
               'mean_network/hidden_1/kernel', 'mean_network/hidden_1/bias',
               'mean_network/output/kernel', 'mean_network/output/bias',
               'log_std_network/log_std_var')
MAX_DEPTH = 3          # hidden layers: 1 to 3 (two run the kernels of PARAM_NAMES above, one and three kernels of their own)


def param_names(depth):
    """Variable names of a policy with `depth` hidden layers, in the reference's creation order (policies/networks/mlp.py:5-62:
    hidden_0 .. hidden_{depth-1}, output; gaussian_mlp_policy.py:55-80: log_std)."""
    names = []
    for i in range(depth):
        names += ['mean_network/hidden_%d/kernel' % i, 'mean_network/hidden_%d/bias' % i]
    return tuple(names) + PARAM_NAMES[4:]
# (obs_dim, action_dim) with policy kernels of their own; every other shape in range runs on the zero-padded kernels
EXACT_SHAPES = ((2, 2), (4, 2), (17, 6))
MAX_OBS_DIM, MAX_ACTION_DIM = 19, 8
# C entry points the algorithms call, by role; a padded shape uses the *_padded sibling of each
POLICY_ENTRIES = ('workspace_bytes', 'forward', 'grad_ex', 'hvp_ragged', 'chain', 'chain_workspace_bytes', 'chain_num_launches')


def _activation_name(fn):
    """'tanh' or 'relu' for a supported hidden_nonlinearity (a name, or a callable such as tf.tanh / tf.nn.relu / torch.relu
    / F.relu, recognised by its __name__), else None."""
    name = 'tanh' if fn is None else (fn if isinstance(fn, str) else getattr(fn, '__name__', None))
    return name if name in ('tanh', 'relu') else None


def _output_activation_name(fn):
    """None (identity) or 'tanh' for a supported output_nonlinearity (None, 'tanh', or a callable named tanh such as tf.tanh /
    torch.tanh); anything else is unsupported and returns False."""
    if fn is None:
        return None
    name = fn if isinstance(fn, str) else getattr(fn, '__name__', None)
    return 'tanh' if name == 'tanh' else False


class MetaGaussianMLPPolicy(object):
    def __init__(self, meta_batch_size, obs_dim, action_dim, name='policy', hidden_sizes=(32, 32), learn_std=True,
                 hidden_nonlinearity='tanh', output_nonlinearity=None, init_std=1., min_std=1e-6, device=None,
                 _skip_param_init=False):
        import torch
        _lib.require_cuda()
        hidden_sizes = tuple(int(h) for h in hidden_sizes)
        if not 1 <= len(hidden_sizes) <= MAX_DEPTH or max(hidden_sizes) > 64 or min(hidden_sizes) < 1:
            raise NotImplementedError("promp_b200 kernels are built for 1 to %d hidden layers of up to 64 units each "
                                      "(got hidden_sizes=%r)" % (MAX_DEPTH, hidden_sizes))
        if not (1 <= int(obs_dim) <= MAX_OBS_DIM and 1 <= int(action_dim) <= MAX_ACTION_DIM):
            raise NotImplementedError("promp_b200 policy kernels take obs_dim in [1, %d] and action_dim in [1, %d] (got %d, %d)"
                                      % (MAX_OBS_DIM, MAX_ACTION_DIM, int(obs_dim), int(action_dim)))
        act = _activation_name(hidden_nonlinearity)
        out = _output_activation_name(output_nonlinearity)
        if act is None or out is False:
            raise NotImplementedError("promp_b200 kernels implement tanh or relu hidden / identity or tanh output non-linearities "
                                      "(got hidden_nonlinearity=%r, output_nonlinearity=%r)"
                                      % (hidden_nonlinearity, output_nonlinearity))
        if not learn_std:
            raise NotImplementedError("learn_std=False is not supported (the reference's meta policy graph requires "
                                      "the log_std variable to be trainable, gaussian_mlp_policy.py:174)")
        self._init_args = dict(meta_batch_size=meta_batch_size, obs_dim=int(obs_dim), action_dim=int(action_dim),
                               name=name, hidden_sizes=hidden_sizes, learn_std=learn_std, init_std=init_std,
                               min_std=min_std, hidden_nonlinearity=act, output_nonlinearity=out)
        self.meta_batch_size = meta_batch_size
        self.obs_dim, self.action_dim, self.name = int(obs_dim), int(action_dim), name
        # The kernels are instantiated for 32 and 64 hidden units; other widths run zero-padded: a padded unit has
        # zero incoming and outgoing weights, so it outputs tanh(0) = relu(0) = 0, receives exactly zero gradient (and zero
        # Hessian-vector product), and therefore stays zero under SGD / Adam / TRPO steps.
        self.hidden_sizes, self.hidden = hidden_sizes, (32 if max(hidden_sizes) <= 32 else 64)
        self.hidden_nonlinearity = act
        self.output_nonlinearity = out        # None (identity) or 'tanh'
        # the `hidden` argument of every policy / rollout kernel call: the width, plus the activation flag for ReLU and the
        # output flag for a tanh mean
        # output flag for a tanh mean, and the depth bits for one or three hidden layers (none for two)
        self.depth = len(hidden_sizes)
        self.hidden_arg = (self.hidden | (_lib.ACT_RELU if act == 'relu' else 0) | (_lib.OUT_TANH if out == 'tanh' else 0)
                           | _lib.hidden_depth(self.depth))
        self.learn_std = learn_std
        self.min_log_std = math.log(min_std)
        self.init_log_std = math.log(init_std)
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._dist = DiagonalGaussian(self.action_dim)
        Hd, names = self.hidden, param_names(self.depth)
        ins = (self.obs_dim,) + hidden_sizes
        shapes = [s for i in range(self.depth) for s in ((ins[i], ins[i + 1]), (ins[i + 1],))]
        self.param_shapes = OrderedDict(zip(names, shapes + [(hidden_sizes[-1], self.action_dim), (self.action_dim,),
                                                             (1, self.action_dim)]))
        self.num_params_logical = int(sum(np.prod(sh) for sh in self.param_shapes.values()))
        # Shapes outside EXACT_SHAPES pad the observation and action axes the same way: W0 gets zero rows up to obs_cap,
        # W2 / b2 / log_std zero columns up to act_cap (promp_policy_layout), and the padded kernels keep them at zero.
        self.padded_dims = (self.obs_dim, self.action_dim) not in EXACT_SHAPES
        if self.padded_dims:
            do_cap, da_cap, _, _ = _lib.policy_layout(self.obs_dim, self.action_dim, self.hidden_arg)
        else:
            do_cap, da_cap = self.obs_dim, self.action_dim
        self.entries = {k: 'promp_policy_' + k + ('_padded' if self.padded_dims else '') for k in POLICY_ENTRIES}
        dev_shapes = (((do_cap, Hd), (Hd,)) + ((Hd, Hd), (Hd,)) * (self.depth - 1)
                      + ((Hd, da_cap), (da_cap,), (1, da_cap)))
        self.num_params = int(sum(np.prod(sh) for sh in dev_shapes))          # device (padded) vector length
        assert self.num_params == _lib.load().promp_num_params(do_cap, da_cap, self.hidden_arg)
        # positions of the logical parameters inside the padded device vector
        idx, off = [], 0
        for (key, shape), dshape in zip(self.param_shapes.items(), dev_shapes):
            grid = np.arange(int(np.prod(dshape))).reshape(dshape) + off
            idx.append(grid[tuple(slice(0, n) for n in shape)].reshape(-1))
            off += int(np.prod(dshape))
        self._pad_index_np = np.concatenate(idx)
        self._log_std_lo = self.num_params - da_cap        # the logical log_std: [lo, lo + action_dim) of the device vector
        self.policy_params_keys = list(names)
        # Xavier-uniform kernels, zero biases, log_std = log(init_std)
        # (policies/networks/mlp.py:12-13, gaussian_mlp_policy.py:64-69); drawn from the numpy global RNG
        flat = []
        for key, shape in self.param_shapes.items():
            if key.endswith('kernel'):
                lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                # unpickling overwrites the parameters right away: do not perturb the seeded global RNG stream for it
                flat.append(np.zeros(int(np.prod(shape))) if _skip_param_init
                            else np.random.uniform(-lim, lim, size=shape).reshape(-1))
            elif key.endswith('bias'):
                flat.append(np.zeros(int(np.prod(shape))))
            else:
                flat.append(np.full(int(np.prod(shape)), self.init_log_std))
        self._pad_index = torch.from_numpy(self._pad_index_np).to(self.device)
        self.theta = torch.zeros(self.num_params, dtype=torch.float32, device=self.device)
        self.theta[self._pad_index] = torch.tensor(np.concatenate(flat), dtype=torch.float32, device=self.device)
        self.theta_tasks = None            # [M, P] post-update parameters
        self._pre_update_mode = True

    # ------------------------------------------------------------------ parameter access
    @property
    def distribution(self):
        return self._dist

    def get_params(self):
        """Reference returns the tf.Variables; here: name -> device tensor (copy of the logical parameters)."""
        return self._unflatten_torch(self.theta[self._pad_index])

    def _unflatten_torch(self, flat):
        out, off = OrderedDict(), 0
        for key, shape in self.param_shapes.items():
            n = int(np.prod(shape))
            out[key] = flat[off:off + n].view(*shape)
            off += n
        return out

    def pad_flat(self, flat):
        """logical flat vector(s) [.., P_logical] (numpy) -> padded device layout [.., P] (numpy)."""
        flat = np.asarray(flat, dtype=np.float32)
        if flat.shape[-1] == self.num_params and self.num_params != self.num_params_logical:
            return flat
        out = np.zeros(flat.shape[:-1] + (self.num_params,), dtype=np.float32)
        out[..., self._pad_index_np] = flat
        return out

    def unpad_flat(self, flat):
        return np.asarray(flat)[..., self._pad_index_np]

    def _unflatten_np(self, flat):
        out, off = OrderedDict(), 0
        for key, shape in self.param_shapes.items():
            n = int(np.prod(shape))
            out[key] = flat[off:off + n].reshape(shape)
            off += n
        return out

    def get_param_values(self):
        """OrderedDict name -> ndarray (policies/base.py:176-184)."""
        return self._unflatten_np(self.unpad_flat(self.theta.detach().cpu().numpy()).copy())

    def set_params(self, policy_params):
        """policies/base.py:186-203; accepts the OrderedDict or a flat vector."""
        import torch
        if isinstance(policy_params, dict):
            assert all(k1 == k2 for k1, k2 in zip(self.param_shapes.keys(), policy_params.keys())), \
                "parameter keys must match with variable"
            flat = np.concatenate([np.asarray(v, dtype=np.float32).reshape(-1) for v in policy_params.values()])
        else:
            flat = np.asarray(policy_params, dtype=np.float32).reshape(-1)
        assert flat.size in (self.num_params_logical, self.num_params)
        self.theta.copy_(torch.from_numpy(self.pad_flat(flat)).to(self.device))

    # ------------------------------------------------------------------ pre / post update bookkeeping
    def switch_to_pre_update(self):
        """policies/base.py:234-240: sampling uses theta for every task (param_stride 0 on the device)."""
        self._pre_update_mode = True
        self.theta_tasks = None

    def update_task_parameters(self, updated_policies_parameters):
        """policies/base.py:262-269.  Accepts a device tensor [M,P] (fast path) or the reference's list of
        M OrderedDicts of numpy arrays."""
        import torch
        if isinstance(updated_policies_parameters, torch.Tensor):
            assert updated_policies_parameters.shape == (self.meta_batch_size, self.num_params)
            self.theta_tasks = updated_policies_parameters
        else:
            assert len(updated_policies_parameters) == self.meta_batch_size
            flat = np.stack([np.concatenate([np.asarray(v, dtype=np.float32).reshape(-1) for v in d.values()])
                             for d in updated_policies_parameters])
            self.theta_tasks = torch.from_numpy(self.pad_flat(flat)).to(self.device)
        self._pre_update_mode = False

    @property
    def policies_params_vals(self):
        if self.theta_tasks is None:
            vals = self.get_param_values()
            return [vals for _ in range(self.meta_batch_size)]
        host = self.unpad_flat(self.theta_tasks.detach().cpu().numpy())
        return [self._unflatten_np(host[i]) for i in range(self.meta_batch_size)]

    def sampling_params(self):
        """(tensor, param_stride, clip_reported_log_std) for the rollout kernel."""
        if self._pre_update_mode or self.theta_tasks is None:
            return self.theta, 0, 1
        return self.theta_tasks, self.num_params, 0

    # ------------------------------------------------------------------ acting (stepwise host API)
    def get_actions(self, observations):
        """policies/meta_gaussian_mlp_policy.py:99-157: list[M] of (E,Do) -> (list[M] of (E,Da),
        list[M][E] of {mean, log_std}).  Forward pass on the device (promp_policy_forward), noise from
        torch's CUDA generator."""
        import torch
        assert len(observations) == self.meta_batch_size
        obs = torch.as_tensor(np.stack([np.asarray(o, dtype=np.float32) for o in observations]), device=self.device)
        M, E = obs.shape[0], obs.shape[1]
        assert obs.shape[2] == self.obs_dim
        params, stride, clip = self.sampling_params()
        mean = torch.empty(M, E, self.action_dim, dtype=torch.float32, device=self.device)
        _lib.call(self.entries['forward'], self.obs_dim, self.action_dim, self.hidden_arg, M, E, _lib.ptr(params), stride,
                  _lib.ptr(obs.contiguous()), _lib.ptr(mean), _lib.stream())
        pm = params.view(-1, self.num_params) if stride else params.view(1, -1).expand(M, -1)
        ls = pm[:, self._log_std_lo:self._log_std_lo + self.action_dim]
        actions = mean + torch.randn_like(mean) * torch.exp(ls).unsqueeze(1)
        rep = torch.clamp(ls, min=self.min_log_std) if clip else ls
        a, mu, rep = actions.cpu().numpy(), mean.cpu().numpy(), rep.cpu().numpy()
        infos = [[dict(mean=mu[m, e], log_std=rep[m]) for e in range(E)] for m in range(M)]
        return [a[m] for m in range(M)], infos

    def get_action(self, observation, task=0):
        obs = np.repeat(np.asarray(observation)[None, None], self.meta_batch_size, axis=0)
        actions, infos = self.get_actions(list(obs))
        return actions[task][0], infos[task][0]

    def reset(self, dones=None):
        pass

    def log_diagnostics(self, paths, prefix=''):
        """gaussian_mlp_policy.py:118-123 (AveragePolicyStd)."""
        phase = getattr(paths[0], 'phase', None) if len(paths) else None
        if phase is not None:
            import torch
            logger.logkv(prefix + 'AveragePolicyStd', float(torch.exp(phase.log_std).mean()))
        else:
            log_stds = np.vstack([path["agent_infos"]["log_std"] for path in paths])
            logger.logkv(prefix + 'AveragePolicyStd', np.mean(np.exp(log_stds)))

    def device_log_terms(self, phase):
        """AveragePolicyStd (gaussian_mlp_policy.py:118-123) as a float64 device vector of length 1."""
        import torch
        return torch.exp(phase.log_std).mean().double().view(1)

    # ------------------------------------------------------------------ pickling (policies/base.py:205-215)
    def __getstate__(self):
        return {'init_args': dict(self._init_args), 'network_params': self.get_param_values()}

    def __setstate__(self, state):
        # no Xavier draw: loading must not consume np.random; a state saved before the activations were stored is tanh with
        # the identity output
        self.__init__(_skip_param_init=True, **state['init_args'])
        self.set_params(state['network_params'])
