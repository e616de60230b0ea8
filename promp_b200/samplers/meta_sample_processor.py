"""MetaSampleProcessor on the GPU.

Mirrors meta_policy_search/samplers/meta_sample_processor.py:6-49 and samplers/base.py:33-173
(constructor arguments, `.baseline`, process_samples(paths_meta_batch, log, log_prefix) -> list of M
dicts with the 8 keys).  All numerics run in promp_process_samples (one CTA per task).  A baseline object without a
`device_kind` (any object with fit / predict, as the reference accepts) is fitted and evaluated on the host; the returns
before it and the GAE, normalisation and statistics after it still run on the device.
"""
import numpy as np

from promp_b200 import _lib
from promp_b200.samplers.device_data import PhaseData, PathsMetaBatch, SamplesData, RaggedPhaseData, RaggedSamplesData
from promp_b200.utils import logger


def _baseline_kind(baseline):
    """The processing kernel's baseline kind, or None for a baseline object whose fit / predict run on the host."""
    return getattr(baseline, 'device_kind', None)


def _coeff_width(baseline_kind, obs_dim):
    return 4 if baseline_kind == _lib.BASELINE_LINEAR_TIME else 2 * obs_dim + 4


def _phase_from_host_paths(paths_meta_batch, device):
    """Upload reference-style host paths (dict of lists of path dicts) into a PhaseData."""
    import torch
    M = len(paths_meta_batch)
    tasks = list(paths_meta_batch.values())
    E = len(tasks[0])
    H = len(tasks[0][0]["rewards"])
    if any(len(paths) != E or any(len(p["rewards"]) != H for p in paths) for paths in tasks):
        return _ragged_phase_from_host_paths(tasks, device)
    obs0 = np.asarray(tasks[0][0]["observations"])
    act0 = np.asarray(tasks[0][0]["actions"])
    Do = obs0.shape[1] if obs0.ndim > 1 else 1
    Da = act0.shape[1] if act0.ndim > 1 else 1
    phase = PhaseData(M, E, H, Do, Da, device)

    def stack(key, d):
        return np.stack([np.concatenate([np.asarray(p[key], dtype=np.float32).reshape(H, d) for p in paths])
                         for paths in tasks])
    phase.obs.copy_(torch.from_numpy(stack("observations", Do)))
    phase.act.copy_(torch.from_numpy(stack("actions", Da)))
    phase.rew.copy_(torch.from_numpy(stack("rewards", 1)[..., 0]))
    phase.done.zero_()
    phase.done.view(M, E, H)[:, :, -1] = 1
    ai = tasks[0][0].get("agent_infos") or {}
    if "mean" in ai:
        phase.mean.copy_(torch.from_numpy(np.stack([np.concatenate(
            [np.asarray(p["agent_infos"]["mean"], dtype=np.float32).reshape(H, Da) for p in paths]) for paths in tasks])))
        phase.log_std.copy_(torch.from_numpy(np.stack(
            [np.asarray(paths[0]["agent_infos"]["log_std"], dtype=np.float32).reshape(H, Da)[0] for paths in tasks])))
    else:
        phase.mean.zero_()
        phase.log_std.zero_()
    return phase


def _ragged_phase_from_host_paths(tasks, device):
    """Variable-length paths (early-terminating envs through the stepwise sampler): padded [M, Nmax] layout + path table."""
    import torch
    if any(len(paths) == 0 for paths in tasks):
        raise ValueError("promp_b200: every task needs at least one completed path")
    obs0 = np.asarray(tasks[0][0]["observations"])
    act0 = np.asarray(tasks[0][0]["actions"])
    Do = obs0.shape[1] if obs0.ndim > 1 else 1
    Da = act0.shape[1] if act0.ndim > 1 else 1
    phase = RaggedPhaseData([[len(p["rewards"]) for p in paths] for paths in tasks], Do, Da, device)
    M, N = phase.M, phase.N

    def stack(key, d, sub=None):
        out = np.zeros((M, N, d), dtype=np.float32)
        for m, paths in enumerate(tasks):
            n = int(phase.n_valid_host[m])
            src = [np.asarray((p[key] if sub is None else p[key][sub]), dtype=np.float32).reshape(-1, d) for p in paths]
            out[m, :n] = np.concatenate(src)
        return out
    phase.obs.copy_(torch.from_numpy(stack("observations", Do)))
    phase.act.copy_(torch.from_numpy(stack("actions", Da)))
    phase.rew.copy_(torch.from_numpy(stack("rewards", 1)[..., 0]))
    done = np.zeros((M, N), dtype=np.uint8)
    for m in range(M):
        done[m, phase.path_off_host[m, 1:phase.n_paths_host[m] + 1] - 1] = 1
    phase.done.copy_(torch.from_numpy(done))
    ai = tasks[0][0].get("agent_infos") or {}
    if "mean" in ai:
        phase.mean.copy_(torch.from_numpy(stack("agent_infos", Da, "mean")))
        phase.log_std.copy_(torch.from_numpy(np.stack(
            [np.asarray(paths[0]["agent_infos"]["log_std"], dtype=np.float32).reshape(-1, Da)[0] for paths in tasks])))
    else:
        phase.log_std.zero_()
    return phase


_WS_CACHE = {}
_WS_KEEP = []       # superseded workspaces stay alive: a captured CUDA graph may still hold their address


def _zeroed_workspace(nbytes, dev):
    """The processing kernel's scratch (arrival tickets + partial Gram blocks): zero-filled ONCE, then left clean by every
    launch, so it is allocated per device (grown on demand) and shared by all phases - launches are serialised on the
    stream.  (A per-phase torch.zeros inside a CUDA-graph capture would replay a fill kernel every iteration.)"""
    import torch
    ws = _WS_CACHE.get(dev)
    if ws is None or ws.numel() * 8 < nbytes:
        ws = torch.zeros((nbytes + 7) // 8 + 64, dtype=torch.float64, device=dev)
        if dev in _WS_CACHE:
            _WS_KEEP.append(_WS_CACHE[dev])
        _WS_CACHE[dev] = ws
    return ws


def run_process_kernel(phase, discount, gae_lambda, reg_coeff, baseline_kind, normalize_adv, positive_adv, given=None):
    """One launch of the processing kernel on `phase`.  baseline_kind BASELINE_GIVEN takes the baseline values from
    `given` (float64 [M, N] device tensor in the phase's sample layout) and writes no coefficients."""
    import torch
    if isinstance(phase, RaggedPhaseData):
        return _run_process_kernel_ragged(phase, discount, gae_lambda, reg_coeff, baseline_kind, normalize_adv, positive_adv,
                                          given)
    M, E, H, Do = phase.M, phase.E, phase.H, phase.obs_dim
    dev = phase.obs.device
    if phase.returns is None:
        phase.returns = torch.empty(M, E * H, dtype=torch.float32, device=dev)
        phase.adv = torch.empty(M, E * H, dtype=torch.float32, device=dev)
        phase.stats = torch.empty(M, 8, dtype=torch.float64, device=dev)
    width = _coeff_width(baseline_kind, Do)
    if phase.coeffs is None or phase.coeffs.shape[1] != width:
        # fully written by the kernel for the linear baselines: no fill launch
        fitted = baseline_kind in (_lib.BASELINE_LINEAR_FEATURE, _lib.BASELINE_LINEAR_TIME)
        phase.coeffs = (torch.empty if fitted else torch.zeros)(M, width, dtype=torch.float64, device=dev)
    nbytes = _lib.load().promp_process_workspace_bytes(M, E, H, Do)
    ws = _zeroed_workspace(nbytes, dev)
    if baseline_kind == _lib.BASELINE_GIVEN:
        _lib.call('promp_process_samples_given', M, E, H, Do, _lib.ptr(phase.obs), _lib.ptr(phase.rew), _lib.ptr(given),
                  float(discount), float(gae_lambda), int(bool(normalize_adv)), int(bool(positive_adv)),
                  _lib.ptr(phase.returns), _lib.ptr(phase.adv), _lib.ptr(phase.stats), _lib.ptr(ws), ws.numel() * 8,
                  _lib.stream())
    else:
        _lib.call('promp_process_samples', M, E, H, Do, _lib.ptr(phase.obs), _lib.ptr(phase.rew), float(discount),
                  float(gae_lambda), float(reg_coeff), int(baseline_kind), int(bool(normalize_adv)), int(bool(positive_adv)),
                  _lib.ptr(phase.returns), _lib.ptr(phase.adv), _lib.ptr(phase.coeffs), _lib.ptr(phase.stats),
                  _lib.ptr(ws), ws.numel() * 8, _lib.stream())
    phase.adj_avg_rewards = None
    phase._explore_adv = None
    phase.invalidate_host()


def _run_process_kernel_ragged(phase, discount, gae_lambda, reg_coeff, baseline_kind, normalize_adv, positive_adv,
                               given=None):
    import torch
    M, Pmax, N, Do = phase.M, phase.E, phase.N, phase.obs_dim
    dev = phase.obs.device
    if phase.returns is None:
        phase.returns = torch.zeros(M, N, dtype=torch.float32, device=dev)
        phase.adv = torch.zeros(M, N, dtype=torch.float32, device=dev)
        phase.stats = torch.zeros(M, 8, dtype=torch.float64, device=dev)
    width = _coeff_width(baseline_kind, Do)
    if phase.coeffs is None or phase.coeffs.shape[1] != width:
        phase.coeffs = torch.zeros(M, width, dtype=torch.float64, device=dev)
    nbytes = _lib.load().promp_process_workspace_bytes_ragged(M, Pmax, N, Do)
    ws = _zeroed_workspace(nbytes, dev)
    if baseline_kind == _lib.BASELINE_GIVEN:
        _lib.call('promp_process_samples_ragged_given', M, Pmax, N, Do, _lib.ptr(phase.obs), _lib.ptr(phase.rew),
                  _lib.ptr(phase.path_off), _lib.ptr(phase.n_paths), _lib.ptr(given), float(discount), float(gae_lambda),
                  int(bool(normalize_adv)), int(bool(positive_adv)), _lib.ptr(phase.returns), _lib.ptr(phase.adv),
                  _lib.ptr(phase.stats), _lib.ptr(ws), ws.numel() * 8, _lib.stream())
    else:
        _lib.call('promp_process_samples_ragged', M, Pmax, N, Do, _lib.ptr(phase.obs), _lib.ptr(phase.rew),
                  _lib.ptr(phase.path_off), _lib.ptr(phase.n_paths), float(discount), float(gae_lambda), float(reg_coeff),
                  int(baseline_kind), int(bool(normalize_adv)), int(bool(positive_adv)), _lib.ptr(phase.returns),
                  _lib.ptr(phase.adv), _lib.ptr(phase.coeffs), _lib.ptr(phase.stats), _lib.ptr(ws), ws.numel() * 8,
                  _lib.stream())
    phase.adj_avg_rewards = None
    phase.invalidate_host()


def _path_offsets(paths):
    """Prefix sums [P+1] int32 of the path lengths len(path["observations"]) (the reference's time index restarts in every
    path, baselines/linear_baseline.py:104, 124)."""
    off = np.zeros(len(paths) + 1, dtype=np.int32)
    off[1:] = np.cumsum([len(p["observations"]) for p in paths])
    return off


def _flat_paths_to_device(paths, dev, with_obs=True):
    """A flat list of (variable-length) host paths -> (obs [n,Do] float32 or None, path_off [P+1] int32, n, Do) on the
    device.  with_obs=False (LinearTimeBaseline): only the path table is uploaded, Do = 1."""
    import torch
    off = _path_offsets(paths)
    if not with_obs:
        return None, torch.from_numpy(off).to(dev), int(off[-1]), 1
    obs = np.concatenate([np.asarray(p["observations"], dtype=np.float32).reshape(int(off[k + 1] - off[k]), -1)
                          for k, p in enumerate(paths)])
    return (torch.from_numpy(np.ascontiguousarray(obs)).to(dev), torch.from_numpy(off).to(dev), int(off[-1]), obs.shape[1])


def fit_baseline_on_paths(paths, target_key, reg_coeff, kind=_lib.BASELINE_LINEAR_FEATURE):
    """LinearBaseline.fit (baselines/linear_baseline.py:55-77) on the device: float64 Gram matrix of the
    LinearFeatureBaseline (kind 1) or LinearTimeBaseline (kind 2) features + ridge solve with the reference's x10-on-NaN
    retry (promp_baseline_fit_ex).  Returns the coefficient vector (2*Do+4 or 4) as a host float64 array."""
    import torch
    _lib.require_cuda()
    assert all(target_key in p.keys() for p in paths)
    dev = torch.device('cuda', torch.cuda.current_device())
    obs, off, n, Do = _flat_paths_to_device(paths, dev, with_obs=kind == _lib.BASELINE_LINEAR_FEATURE)
    target = torch.from_numpy(np.concatenate([np.asarray(p[target_key], dtype=np.float64).reshape(-1) for p in paths])).to(dev)
    assert target.numel() == n, "targets and observations must have the same length"
    coeffs = torch.empty(_coeff_width(kind, Do), dtype=torch.float64, device=dev)
    ws = _zeroed_workspace(_lib.load().promp_baseline_fit_workspace_bytes(len(paths), n, Do), dev)
    _lib.call('promp_baseline_fit_ex', int(kind), len(paths), n, Do, _lib.ptr(obs), _lib.ptr(target), _lib.ptr(off),
              float(reg_coeff), _lib.ptr(coeffs), None, _lib.ptr(ws), ws.numel() * 8, _lib.stream())
    return coeffs.cpu().numpy()


def predict_baseline_on_path(path, coeffs, kind=_lib.BASELINE_LINEAR_FEATURE):
    """LinearBaseline.predict (baselines/linear_baseline.py:17-33) on the device (promp_baseline_predict_ex)."""
    import torch
    _lib.require_cuda()
    dev = torch.device('cuda', torch.cuda.current_device())
    obs, off, n, Do = _flat_paths_to_device([path], dev, with_obs=kind == _lib.BASELINE_LINEAR_FEATURE)
    w = torch.from_numpy(np.ascontiguousarray(np.asarray(coeffs, dtype=np.float64))).to(dev)
    assert w.numel() == _coeff_width(kind, Do), "coefficient vector does not match the baseline's features"
    out = torch.empty(n, dtype=torch.float64, device=dev)
    _lib.call('promp_baseline_predict_ex', int(kind), 1, n, Do, _lib.ptr(obs), _lib.ptr(off), _lib.ptr(w), _lib.ptr(out),
              _lib.stream())
    return out.cpu().numpy()


def _host_task_paths(phase, m):
    """Task m of a processed phase as the reference's path dicts (meta_sampler.py:116-123) plus 'returns'
    (samplers/base.py:103-104), from one host copy of the phase's tensors.  Arrays are float32, as the phase stores them."""
    if isinstance(phase, RaggedPhaseData):
        bounds = phase.path_off_host[m][:int(phase.n_paths_host[m]) + 1]
    else:
        bounds = np.arange(phase.E + 1) * phase.H
    obs, act, rew, ret, mean = (phase.host(k)[m] for k in ('obs', 'act', 'rew', 'returns', 'mean'))
    log_std = phase.host('log_std')[m]
    info = phase.host('info') if phase.info_keys else None
    paths = []
    for k in range(len(bounds) - 1):
        s = slice(int(bounds[k]), int(bounds[k + 1]))
        paths.append(dict(observations=obs[s], actions=act[s], rewards=rew[s], returns=ret[s],
                          env_infos={key: info[i, m, s] for i, key in enumerate(phase.info_keys)},
                          agent_infos=dict(mean=mean[s], log_std=np.broadcast_to(log_std, (s.stop - s.start, phase.act_dim)))))
    return paths


class MetaSampleProcessor(object):
    def __init__(self, baseline, discount=0.99, gae_lambda=1, normalize_adv=False, positive_adv=False):
        assert 0 <= discount <= 1.0, 'discount factor must be in [0,1]'
        assert 0 <= gae_lambda <= 1.0, 'gae_lambda must be in [0,1]'
        assert hasattr(baseline, 'fit') and hasattr(baseline, 'predict')
        self.baseline = baseline
        self.discount = discount
        self.gae_lambda = gae_lambda
        self.normalize_adv = normalize_adv
        self.positive_adv = positive_adv

    def process_phase(self, phase):
        """Run the processing kernel on a PhaseData.  With a device baseline (`device_kind`) nothing leaves the device;
        any other baseline object goes through _process_phase_host_baseline."""
        kind = _baseline_kind(self.baseline)
        if kind is None:
            return self._process_phase_host_baseline(phase)
        run_process_kernel(phase, self.discount, self.gae_lambda, getattr(self.baseline, '_reg_coeff', 1e-5),
                           kind, self.normalize_adv, self.positive_adv)
        if hasattr(self.baseline, '_coeffs') and kind in (_lib.BASELINE_LINEAR_FEATURE, _lib.BASELINE_LINEAR_TIME):
            # the reference's baseline object holds the last fit = the last task's (baselines/linear_baseline.py:55-77): a lazy
            # view of the device buffer, fetched on demand (a replayed CUDA graph rewrites the same buffer every iteration)
            self.baseline._lazy_coeffs = (phase, phase.M - 1)
            self.baseline._coeffs = _LazyCoeffs(phase)
        return phase

    def _process_phase_host_baseline(self, phase):
        """A baseline with fit / predict but no device kind (samplers/base.py:99-108 asserts nothing more):
          1. the ZERO kind computes the discounted returns on the device (the same returns the final pass writes);
          2. for tasks m = 0..M-1 in order, the task's path dicts, 'returns' included, go to baseline.fit(paths,
             target_key='returns'), then baseline.predict(path) runs for each path in order - the reference's sequence, so
             the object is left fitted on the last task.  The arrays are float32 (observations, rewards and returns as
             the phase stores them), not the reference's float64 returns;
          3. every prediction goes up in one H2D copy and the GIVEN kind runs GAE, normalisation and the statistics."""
        import torch
        run_process_kernel(phase, self.discount, self.gae_lambda, 0.0, _lib.BASELINE_ZERO, self.normalize_adv,
                           self.positive_adv)
        values = np.zeros((phase.M, phase.N), dtype=np.float64)
        for m in range(phase.M):
            paths = _host_task_paths(phase, m)
            self.baseline.fit(paths, target_key='returns')
            n = 0
            for p in paths:
                L = len(p['rewards'])
                values[m, n:n + L] = np.asarray(self.baseline.predict(p), dtype=np.float64).reshape(L)
                n += L
        given = torch.from_numpy(values).to(phase.obs.device)
        run_process_kernel(phase, self.discount, self.gae_lambda, 0.0, _lib.BASELINE_GIVEN, self.normalize_adv,
                           self.positive_adv, given=given)
        return phase

    def compute_adj_avg_rewards(self, phase, allreduce=None):
        """samples_data['adj_avg_rewards'] (meta_sample_processor.py:40-44), computed on first access."""
        import torch
        st = phase.stats[:, 5:7].sum(0)
        n_total = float(phase.n_valid_host.sum()) if isinstance(phase, RaggedPhaseData) else float(phase.M * phase.N)
        cnt = torch.tensor([n_total], dtype=torch.float64, device=st.device)
        vec = torch.cat([st, cnt])
        if allreduce is not None:
            allreduce(vec)
        s, s2, n = [float(x) for x in vec.cpu()]
        mean = s / n
        std = max(s2 / n - mean * mean, 0.0) ** 0.5
        phase.adj_avg_rewards = torch.empty_like(phase.rew)
        _lib.call('promp_adj_avg_rewards', phase.rew.numel(), _lib.ptr(phase.rew), mean, std,
                  _lib.ptr(phase.adj_avg_rewards), _lib.stream())
        phase._host.pop('adj_avg_rewards', None)

    def process_samples(self, paths_meta_batch, log=False, log_prefix=''):
        """meta_sample_processor.py:8-49."""
        import torch
        assert isinstance(paths_meta_batch, dict), 'paths must be a dict'
        assert self.baseline, 'baseline must be specified'
        phase = getattr(paths_meta_batch, 'phase', None)
        if phase is None:
            _lib.require_cuda()
            phase = _phase_from_host_paths(paths_meta_batch, torch.device('cuda', torch.cuda.current_device()))
        self.process_phase(phase)
        cls = RaggedSamplesData if isinstance(phase, RaggedPhaseData) else SamplesData
        samples = [cls(phase, m, self) for m in range(phase.M)]
        self._log_path_stats(phase, log, log_prefix)
        return samples

    PATH_STAT_KEYS = ('AverageDiscountedReturn', 'AverageReturn', 'NumTrajs', 'StdReturn', 'MaxReturn', 'MinReturn')

    def device_log_terms(self, phase):
        """The six path statistics of samplers/base.py:135-149 as one float64 device vector (no host sync):
        used by the CUDA-graph Trainer, which reads all logged scalars back with a single D2H copy."""
        import torch
        st = phase.stats
        n = float(phase.total_paths) if isinstance(phase, RaggedPhaseData) else float(phase.M * phase.E)
        s = st[:, :3].sum(0)
        mean_g = s[1] / n
        std = torch.sqrt(torch.clamp(s[2] / n - mean_g * mean_g, min=0.0))
        return torch.stack([s[0] / n, mean_g, torch.full_like(mean_g, n), std, st[:, 3].max(), st[:, 4].min()])

    def _log_path_stats(self, phase, log=False, log_prefix=''):
        """samplers/base.py:135-149 from the per-task sums the kernel wrote (one small D2H)."""
        if not log:
            return
        st = phase.host('stats')
        n = phase.total_paths if isinstance(phase, RaggedPhaseData) else phase.M * phase.E
        sR0, sG, sG2 = st[:, 0].sum(), st[:, 1].sum(), st[:, 2].sum()
        mean_g = sG / n
        if log == 'reward':
            logger.logkv(log_prefix + 'AverageReturn', mean_g)
        elif log == 'all' or log is True:
            logger.logkv(log_prefix + 'AverageDiscountedReturn', sR0 / n)
            logger.logkv(log_prefix + 'AverageReturn', mean_g)
            logger.logkv(log_prefix + 'NumTrajs', n)
            logger.logkv(log_prefix + 'StdReturn', float(np.sqrt(max(sG2 / n - mean_g * mean_g, 0.0))))
            logger.logkv(log_prefix + 'MaxReturn', st[:, 3].max())
            logger.logkv(log_prefix + 'MinReturn', st[:, 4].min())


class _LazyCoeffs(object):
    """Stands in for baseline._coeffs until someone needs the numbers (avoids a D2H per phase)."""

    def __init__(self, phase):
        self._phase = phase
        self._val = None

    def _get(self):
        if self._val is None:
            self._val = self._phase.host('coeffs')[-1].copy()
        return self._val

    def __array__(self, dtype=None, copy=None):
        v = self._get()
        return v.astype(dtype) if dtype is not None else v

    def __len__(self):
        return len(self._get())

    def __getitem__(self, i):
        return self._get()[i]

    def dot(self, other):
        return self._get().dot(other)
