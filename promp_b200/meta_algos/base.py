"""MAMLAlgo on the GPU (ref: meta_policy_search/meta_algos/base.py:85-313).

The reference builds a TF graph with M replicated per-task sub-graphs and lets tf.gradients
differentiate through the inner SGD step.  Here the same quantities are produced by three kernels:

  forward chain   theta_{s+1,i} = theta_{s,i} - alpha * grad surr_s,i(theta_{s,i})   promp_policy_grad (+SGD)
  outer gradient  v_i = grad_{theta'} L_i(theta_{S-1,i})                             promp_policy_grad
  backward chain  v_i <- v_i - alpha * H_s,i v_i + c_s * grad KL_s,i                 promp_policy_hvp
  meta-gradient   g = (1/M) sum_i v_i   (+ all-reduce over ranks)                    promp_reduce_tasks

which is exactly d/dtheta of the meta objective for any number of inner steps (the backward chain
is the transpose of d theta_{s+1} / d theta_s = I - alpha H_s).

trainable_inner_step_size=True (Meta-SGD, Li et al. 2017; ref base.py:98, 210, 303-313): alpha is a vector [P] in the
policy's device layout, shared by every task and inner step, that starts at inner_lr and is trained with theta:
  forward chain   theta_{s+1,i} = theta_{s,i} - alpha * g_{s,i}                      (alpha: PolicyStage.step_size)
  backward chain  v_i <- v_i - H_s,i (alpha * v_i) + c_s * grad KL_s,i
  alpha gradient  -(1/M) sum_i sum_s v_{s+1,i} * g_{s,i}   (v_{s+1,i}: the vector entering the HVP stage of step s)
"""
import ctypes
import os

import numpy as np

from promp_b200 import _lib
from promp_b200.samplers.device_data import SamplesData, PhaseData, RaggedSamplesData
from promp_b200.utils.dist import allreduce_sum_, world_size  # noqa: F401


class MAMLAlgo(object):
    """
    Args:
        policy (MetaGaussianMLPPolicy), inner_lr, meta_batch_size, num_inner_grad_steps,
        trainable_inner_step_size (bool): learn one inner step size per policy parameter (Meta-SGD) with the outer optimizer
    """
    inner_obj_kind = _lib.OBJ_RATIO
    CHAIN_MAX_STAGES = 6          # promp_policy_chain's stage limit
    MAX_INNER_GRAD_STEPS = 6      # promp_meta_loss_terms / promp_adapt_kl_coeff take at most 7 sampling phases
    STATS_SLOTS = 16              # per-evaluation stats buffers kept per (S, M), see _stats_rows

    def __init__(self, policy, inner_lr=0.1, meta_batch_size=20, num_inner_grad_steps=1,
                 trainable_inner_step_size=False):
        assert hasattr(policy, 'sampling_params'), "policy must be a promp_b200 MetaGaussianMLPPolicy"
        assert type(num_inner_grad_steps) and num_inner_grad_steps >= 0
        if num_inner_grad_steps > self.MAX_INNER_GRAD_STEPS:
            raise ValueError("num_inner_grad_steps=%d: at most %d inner gradient steps are supported (the device loss-term and "
                             "KL-coefficient kernels take up to %d sampling phases)"
                             % (num_inner_grad_steps, self.MAX_INNER_GRAD_STEPS, self.MAX_INNER_GRAD_STEPS + 1))
        assert type(meta_batch_size) == int
        self.policy = policy
        self.inner_lr = float(inner_lr)
        self.meta_batch_size = meta_batch_size
        self.num_inner_grad_steps = num_inner_grad_steps
        self.trainable_inner_step_size = bool(trainable_inner_step_size)
        # alpha [P] on the device (padded layout included), trained by the outer optimizer; None = the scalar inner_lr
        self.alpha = None
        if self.trainable_inner_step_size:
            import torch
            self.alpha = torch.full((policy.num_params,), self.inner_lr, dtype=torch.float32, device=policy.device)
        self._optimization_keys = None
        self._ws = None
        self._ws_chain = None
        self._stats_ring = {}
        # the gradient chain of a meta-objective evaluation as ONE dataflow launch (promp_policy_chain) or as one launch per stage
        self.use_chain = os.environ.get('PROMP_B200_CHAIN', '1') != '0'

    @property
    def step_sizes(self):
        """The inner step sizes as the reference's `step_sizes` dict: parameter key -> numpy array of the parameter's shape
        (inner_lr everywhere unless trainable_inner_step_size)."""
        p = self.policy
        flat = self.alpha.cpu().numpy() if self.alpha is not None else np.full(p.num_params, self.inner_lr, np.float32)
        return p._unflatten_np(p.unpad_flat(flat).copy())

    # ------------------------------------------------------------------------------------ helpers
    def _workspace(self, N):
        import torch
        p = self.policy
        need = getattr(_lib.load(), p.entries['workspace_bytes'])(self.meta_batch_size, N, p.obs_dim, p.action_dim, p.hidden_arg)
        if self._ws is None or self._ws.numel() * 4 < need:
            self._ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device=p.device)   # counters start at zero
        return self._ws

    def _stats_rows(self, S):
        """The [S, M, 4] float32 stats buffer of one evaluation (row s = launch s), taken in turn from STATS_SLOTS buffers
        that are allocated and zero-filled together on first use, like the workspaces.  The kernels write columns 0-2 and
        never column 3, which therefore stays zero: an evaluation's stats are defined in full without a fill per evaluation
        (a captured iteration replays no fill).  A buffer is handed out again STATS_SLOTS evaluations later; every consumer
        reads its rows on the stream before that (promp_meta_loss_terms, the loss-term sums, the tests' clones)."""
        import torch
        M = self.meta_batch_size
        ring = self._stats_ring.get(S)
        if ring is None:
            ring = self._stats_ring[S] = [torch.zeros(self.STATS_SLOTS, S, M, 4, dtype=torch.float32, device=self.policy.device), 0]
        buf = ring[0][ring[1]]
        ring[1] = (ring[1] + 1) % self.STATS_SLOTS
        return buf

    def _phase_of(self, samples):
        """samples: list (len M) of per-task dicts -> PhaseData on the device."""
        import torch
        assert len(samples) == self.meta_batch_size
        first = samples[0]
        if isinstance(first, (SamplesData, RaggedSamplesData)) and \
                all(isinstance(s, (SamplesData, RaggedSamplesData)) and s.phase is first.phase for s in samples):
            return first.phase
        # reference-style numpy dicts: upload (ref _extract_input_dict, base.py:245-280)
        p = self.policy
        N = len(first['advantages'])
        E = 1
        phase = PhaseData(self.meta_batch_size, E, N, p.obs_dim, p.action_dim, p.device)

        def up(key, sub=None):
            arr = np.stack([np.asarray(s[key] if sub is None else s[key][sub], dtype=np.float32) for s in samples])
            return torch.from_numpy(np.ascontiguousarray(arr)).to(p.device)
        phase.obs = up('observations').reshape(self.meta_batch_size, N, p.obs_dim)
        phase.act = up('actions').reshape(self.meta_batch_size, N, p.action_dim)
        phase.adv = up('advantages').reshape(self.meta_batch_size, N)
        phase.mean = up('agent_infos', 'mean').reshape(self.meta_batch_size, N, p.action_dim)
        phase.log_std_full = up('agent_infos', 'log_std').reshape(self.meta_batch_size, N, p.action_dim)
        if 'adj_avg_rewards' in first:
            # E-MAML (trpo_maml.py:137-144 / vpg_maml.py:137-144) only uses mean_n adj_avg_rewards_i: keep that per task
            c = np.asarray([np.mean(np.asarray(s['adj_avg_rewards'], dtype=np.float64)) for s in samples], dtype=np.float32)
            phase.adj_avg_rewards_mean = torch.from_numpy(c).to(p.device)
        return phase

    def _grad(self, phase, params, stride, obj_kind, obj_scale=1.0, clip_eps=0.0, kl_coeff=0.0, clip_log_std=0,
              grad=None, out_params=None, sgd_lr=0.0, stats=None, produce=None, reuse=None, adv=None):
        """One promp_policy_grad launch.  produce / reuse = (flag int32[1], theta copy [P]): the launch re-use protocol of
        promp_policy_grad_ex (the _adapt launch produces, the identical inner pass of the first Adam epoch re-uses).
        adv: the weights in place of phase.adv (OBJ_EXPLORE: the per-task E-MAML coefficient [M])."""
        p = self.policy
        ws = self._workspace(phase.N)
        full = getattr(phase, 'log_std_full', None)
        old_ls, per_sample = (full, 1) if full is not None else (phase.log_std, 0)
        n_valid = getattr(phase, 'n_valid', None)           # variable-length paths: per-task sample counts
        skip = (_lib.ptr(reuse[0]), _lib.ptr(reuse[1])) if reuse is not None else (None, None)
        prod = (_lib.ptr(produce[0]), _lib.ptr(produce[1])) if produce is not None else (None, None)
        _lib.call(p.entries['grad_ex'], p.obs_dim, p.action_dim, p.hidden_arg, self.meta_batch_size, phase.N, _lib.ptr(n_valid),
                  _lib.ptr(params), stride, _lib.ptr(phase.obs), _lib.ptr(phase.act), _lib.ptr(phase.adv if adv is None else adv),
                  _lib.ptr(phase.mean), _lib.ptr(old_ls), per_sample, obj_kind, float(obj_scale), float(clip_eps),
                  float(kl_coeff), int(clip_log_std), float(p.min_log_std), _lib.ptr(grad), _lib.ptr(out_params),
                  float(sgd_lr), _lib.ptr(stats), skip[0], skip[1], prod[0], prod[1], _lib.ptr(ws), ws.numel() * 4, _lib.stream())

    def _stage(self, kind, phase, params, stride, obj_kind, obj_scale=1.0, clip_eps=0.0, kl_coeff=0.0, clip_log_std=0, grad=None,
               out_params=None, sgd_lr=0.0, vec=None, out=None, stats=None, kl_coeff_dev=None, adv=None):
        """One promp_policy_stage (kind 0: the arguments of _grad, kind 1: those of _hvp).  With trainable step sizes, the SGD
        step of a gradient stage with out_params and every HVP stage use alpha (self.alpha) in place of inner_lr."""
        full = getattr(phase, 'log_std_full', None)
        old_ls, per_sample = (full, 1) if full is not None else (phase.log_std, 0)
        st = _lib.PolicyStage()
        st.kind, st.N, st.n_valid = kind, phase.N, _lib.ptr(getattr(phase, 'n_valid', None))
        st.params, st.param_stride = _lib.ptr(params), stride
        st.obs, st.act, st.adv, st.old_mean, st.old_log_std = (_lib.ptr(phase.obs), _lib.ptr(phase.act),
                                                               _lib.ptr(phase.adv if adv is None else adv), _lib.ptr(phase.mean),
                                                               _lib.ptr(old_ls))
        st.ls_per_sample, st.obj_kind, st.obj_scale, st.clip_eps = per_sample, obj_kind, float(obj_scale), float(clip_eps)
        st.kl_coeff, st.clip_log_std = float(kl_coeff), int(clip_log_std)
        st.grad, st.out_params, st.sgd_lr = _lib.ptr(grad), _lib.ptr(out_params), float(sgd_lr)
        st.inner_lr, st.vec, st.out, st.stats = float(self.inner_lr), _lib.ptr(vec), _lib.ptr(out), _lib.ptr(stats)
        st.kl_coeff_dev = _lib.ptr(kl_coeff_dev)      # optional device-resident multiplier of kl_coeff
        if self.alpha is not None and (kind == 1 or out_params is not None):
            st.step_size = _lib.ptr(self.alpha)
            st.inner_lr = 1.0                          # HVP stage: vec - H (alpha * vec)
        return st

    def _run_chain(self, stages, reuse=None):
        """promp_policy_chain over a list of PolicyStage (all buffers must stay alive until the launch has run).  A list longer
        than CHAIN_MAX_STAGES (three or more inner steps) runs as consecutive launches of at most CHAIN_MAX_STAGES stages on
        one stream: stream order is the dependency between them, and each launch leaves the shared workspace's control
        words zero.  The launch re-use pointers belong to stage 0, so only the first launch gets them."""
        import torch
        p = self.policy
        pieces = [(_lib.PolicyStage * len(part))(*part)
                  for part in (stages[i:i + self.CHAIN_MAX_STAGES] for i in range(0, len(stages), self.CHAIN_MAX_STAGES))]
        need = 0
        for arr in pieces:
            n = getattr(_lib.load(), p.entries['chain_workspace_bytes'])(p.obs_dim, p.action_dim, p.hidden_arg, self.meta_batch_size,
                                                                         len(arr), ctypes.cast(arr, ctypes.c_void_p))
            if n < 0:
                raise _lib.PrompLibraryError(p.entries['chain_workspace_bytes'] + ": " + _lib.last_error())
            need = max(need, n)
        if self._ws_chain is None or self._ws_chain.numel() * 4 < need:
            self._ws_chain = torch.zeros((need + 3) // 4, dtype=torch.int32, device=p.device)   # control words start at zero
        ws = self._ws_chain
        skip = (_lib.ptr(reuse[0]), _lib.ptr(reuse[1])) if reuse is not None else (None, None)
        for i, arr in enumerate(pieces):
            _lib.call(p.entries['chain'], p.obs_dim, p.action_dim, p.hidden_arg, self.meta_batch_size, float(p.min_log_std),
                      len(arr), ctypes.cast(arr, ctypes.c_void_p), skip[0] if i == 0 else None, skip[1] if i == 0 else None,
                      _lib.ptr(ws), ws.numel() * 4, _lib.stream())

    def _hvp(self, phase, params, stride, vec, out, kl_coeff, clip_log_std, stats=None):
        p = self.policy
        ws = self._workspace(phase.N)
        full = getattr(phase, 'log_std_full', None)
        old_ls, per_sample = (full, 1) if full is not None else (phase.log_std, 0)
        n_valid = getattr(phase, 'n_valid', None)           # NULL: every task has N valid samples
        _lib.call(p.entries['hvp_ragged'], p.obs_dim, p.action_dim, p.hidden_arg, self.meta_batch_size, phase.N, _lib.ptr(n_valid),
                  _lib.ptr(params), stride, _lib.ptr(phase.obs), _lib.ptr(phase.act), _lib.ptr(phase.adv),
                  _lib.ptr(phase.mean), _lib.ptr(old_ls), per_sample, self.inner_obj_kind, float(self.inner_lr),
                  float(kl_coeff), int(clip_log_std), float(p.min_log_std), _lib.ptr(vec), _lib.ptr(out),
                  _lib.ptr(stats), _lib.ptr(ws), ws.numel() * 4, _lib.stream())

    # ------------------------------------------------------------------------------------ inner step
    def _adapt_launch(self, phase):
        """theta_i' = theta_i - alpha * grad surr_i(theta_i) for all tasks in one launch (MAMLAlgo._adapt, base.py:217-242).  From
        the shared pre-update parameters the launch also leaves what the first Adam epoch's identical inner pass needs to
        skip itself (promp_policy_grad_ex): its outputs (gradient, theta', stats row 0 of a [S, M, 4] buffer), a copy of the
        parameters it used and the no-clip flag."""
        import torch
        p = self.policy
        params, stride, _ = p.sampling_params()
        M, P = self.meta_batch_size, p.num_params
        grad = torch.empty(M, P, dtype=torch.float32, device=p.device)
        new = torch.empty(M, P, dtype=torch.float32, device=p.device)
        produce, stats = None, None
        self._adapt_cache = None
        if self.alpha is not None:
            # per-parameter step sizes go through the stage path; no launch re-use (the first Adam epoch recomputes stage 0)
            st = self._stage(0, phase, params, stride, self.inner_obj_kind, grad=grad, out_params=new)
            self._run_chain([st])
            self.last_inner_grad = grad
            p.update_task_parameters(new)
            return
        if stride == 0 and params is p.theta and getattr(phase, 'n_valid', None) is None:
            if getattr(self, '_reuse_bufs', None) is None:
                self._reuse_bufs = (torch.zeros(1, dtype=torch.int32, device=p.device),
                                    torch.empty(P, dtype=torch.float32, device=p.device))
            stats_all = self._stats_rows(self.num_inner_grad_steps + 1)
            produce, stats = self._reuse_bufs, stats_all[0]
            self._adapt_cache = dict(phase=phase, adv=phase.adv, gen=getattr(phase, 'generation', 0), grad=grad, new=new,
                                     stats_all=stats_all)
        # the adapt graph is fed parameter placeholders: no log_std clip (gaussian_mlp_policy.py:164-182)
        self._grad(phase, params, stride, self.inner_obj_kind, grad=grad, out_params=new, sgd_lr=self.inner_lr, stats=stats,
                   produce=produce)
        self.last_inner_grad = grad
        p.update_task_parameters(new)

    def adapt_phase(self, phase):
        """_adapt on a PhaseData directly (no per-task dict views): used by the CUDA-graph Trainer."""
        self._adapt_launch(phase)

    def _adapt(self, samples):
        """MAMLAlgo._adapt (base.py:217-242): theta_i' = theta_i - alpha * grad surr_i(theta_i), all tasks
        in one launch, result stays on the device and becomes the sampling policy."""
        assert len(samples) == self.meta_batch_size
        self._adapt_launch(self._phase_of(samples))

    # ------------------------------------------------------------------------------------ meta objective
    def _meta_pass(self, theta, phases, outer_obj_kind, clip_eps, inner_kl_coeffs, want_grad, outer_kl_coeff=0.0,
                   outer_obj_scale=1.0, reduce=True, inner_kl_coeffs_dev=None, explore=None):
        """One evaluation of the meta objective (and optionally its gradient) at `theta` [P].

        Returns dict(grad=[P] or None (local sum over tasks / M_global, NOT yet all-reduced),
                     surr=[M] outer surrogate per task, outer_kl=[M], inner_kl=[S-1, M]).
        reduce=False leaves the per-task gradients in out['grad_tasks'] [M, P] for the fused reduce + all-reduce + Adam
        kernel (promp_meta_update) and skips promp_reduce_tasks.
        Trainable step sizes: out['sgd_pairs'] = [(v_{s+1}, g_s)] per inner step s (the direction entering HVP stage s and the
        inner gradient of stage s, both [M, P]) for promp_meta_update_sgd, and with reduce=True out['grad'] is the [2P]
        gradient [theta; alpha].
        explore: the E-MAML coefficient c [M] (device) or None.  The exploration term -c_m * mean logp_theta(a|x) on the
        phase-0 data (trpo_maml.py:137-144) is then one more gradient stage (OBJ_EXPLORE at theta, clipped log_std) of the
        chain; out['explore'] = its value per task [M], and its gradient is summed into out['grad'] by the same reduction."""
        import torch
        p = self.policy
        M, P, S = self.meta_batch_size, p.num_params, len(phases)
        dev = p.device
        assert explore is None or reduce, "the exploration gradient is added by promp_reduce_tasks2 (reduce=True)"
        x_stats = torch.empty(M, 4, dtype=torch.float32, device=dev) if explore is not None else None
        x_grad = torch.empty(M, P, dtype=torch.float32, device=dev) if explore is not None and want_grad else None

        def reduced(v):
            flat = torch.empty(P if self.alpha is None else 2 * P, dtype=torch.float32, device=dev)
            if self.alpha is not None:       # the alpha half first (task_grads NULL: promp_reduce_tasks_sgd writes only it)
                lam, g = _lib.ptr_array([a for a, _ in pairs]), _lib.ptr_array([b for _, b in pairs])   # kept alive here
                _lib.call('promp_reduce_tasks_sgd', M, P, None, len(pairs), lam, g, 1.0 / (M * world_size()), _lib.ptr(flat),
                          _lib.stream())
            if x_grad is None:
                _lib.call('promp_reduce_tasks', M, P, _lib.ptr(v), 1.0 / (M * world_size()), _lib.ptr(flat), _lib.stream())
            else:
                _lib.call('promp_reduce_tasks2', M, P, _lib.ptr(v), _lib.ptr(x_grad), 1.0 / (M * world_size()), _lib.ptr(flat),
                          _lib.stream())
            return flat

        def explore_launch():
            self._grad(phases[0], theta, 0, _lib.OBJ_EXPLORE, clip_log_std=1, grad=x_grad, stats=x_stats, adv=explore)
        cur, stride, clip = theta, 0, 1              # step 0 = distribution_info_sym(params=None): clipped log_std
        chain = []
        pairs = []                                   # trainable step sizes: (v_{s+1}, g_s) per inner step
        trainable = self.alpha is not None
        # The inner pass at step 0 repeats the _adapt launch as long as theta has not been updated since (first Adam epoch,
        # "loss before" passes): aim it at the SAME output buffers and let the kernel skip itself after verifying on the
        # device that the parameters are bit-identical and the step-0 log_std clip is inactive.  Host-side conditions: same
        # phase object / advantage tensor / data generation, shared parameters, same number of inner steps; only the FIRST pass
        # after _adapt takes this route.
        cache = getattr(self, '_adapt_cache', None)
        reuse0 = (cache is not None and S >= 2 and theta is p.theta and cache['phase'] is phases[0]
                  and cache['adv'] is phases[0].adv and cache['gen'] == getattr(phases[0], 'generation', 0)
                  and cache['stats_all'].shape[0] == S)
        if reuse0:
            stats_all = cache['stats_all']
            self._adapt_cache = None          # one consumer: later passes (updated theta) use their own buffers
        else:
            stats_all = self._stats_rows(S)   # one stats buffer per evaluation (no fills, no copies): row s = launch s
        if inner_kl_coeffs_dev is not None and not self.use_chain:
            # the stand-alone entry points take the coefficient by value: read the device vector back (eager diagnostics only)
            host = inner_kl_coeffs_dev.cpu().numpy()
            inner_kl_coeffs = [float(np.float32(sc) * np.float32(c)) for sc, c in zip(inner_kl_coeffs, host)]
            inner_kl_coeffs_dev = None
        if (self.use_chain or trainable) and (S >= 2 or want_grad):
            # the whole chain - inner gradients + SGD steps, outer gradient, backward Hessian-vector chain - as ONE launch
            stages = []
            for s in range(S - 1):
                if s == 0 and reuse0:
                    g, nxt = cache['grad'], cache['new']
                else:
                    g = torch.empty(M, P, dtype=torch.float32, device=dev)
                    nxt = torch.empty(M, P, dtype=torch.float32, device=dev)
                stages.append(self._stage(0, phases[s], cur, stride, self.inner_obj_kind, clip_log_std=clip, grad=g, out_params=nxt,
                                          sgd_lr=self.inner_lr, stats=stats_all[s]))
                chain.append((cur, stride, clip, g))
                cur, stride, clip = nxt, P, 0
            v = torch.empty(M, P, dtype=torch.float32, device=dev) if want_grad else None
            stages.append(self._stage(0, phases[-1], cur, stride, outer_obj_kind, obj_scale=outer_obj_scale, clip_eps=clip_eps,
                                      kl_coeff=outer_kl_coeff, clip_log_std=clip, grad=v, stats=stats_all[S - 1]))
            if want_grad:
                for s in range(S - 2, -1, -1):
                    prm, strd, clp, _ = chain[s]
                    # out-of-place: a direction vector nothing in the launch writes may be read through the read-only path
                    v_out = torch.empty(M, P, dtype=torch.float32, device=dev)
                    stages.append(self._stage(1, phases[s], prm, strd, self.inner_obj_kind, kl_coeff=inner_kl_coeffs[s],
                                              clip_log_std=clp, vec=v, out=v_out,
                                              kl_coeff_dev=None if inner_kl_coeffs_dev is None else inner_kl_coeffs_dev[s:s + 1]))
                    chain.append(v)       # the stage list holds raw pointers: keep every buffer alive until the launch is enqueued
                    if trainable:
                        pairs.insert(0, (v, chain[s][3]))
                    v = v_out
            if explore is not None:
                # last stage, waits for no other: in the dataflow kernel it fills the tail of the backward chain
                stages.append(self._stage(0, phases[0], theta, 0, _lib.OBJ_EXPLORE, clip_log_std=1, grad=x_grad, stats=x_stats,
                                          adv=explore))
            if trainable and not self.use_chain:
                for st in stages:                      # one launch per stage
                    self._run_chain([st])
            else:
                self._run_chain(stages, reuse=self._reuse_bufs if reuse0 else None)
            out = dict(surr=stats_all[S - 1, :, 0], outer_kl=stats_all[S - 1, :, 1], inner_kl=stats_all[:S - 1, :, 1],
                       stats_all=stats_all, grad=None)
            if trainable and want_grad:
                out['sgd_pairs'] = pairs
            if x_stats is not None:
                out['explore'] = x_stats[:, 0]
            if want_grad:
                if reduce:
                    out['grad'] = reduced(v)
                else:
                    out['grad_tasks'] = v
            return out
        for s in range(S - 1):
            if s == 0 and reuse0:
                g, nxt = cache['grad'], cache['new']
                self._grad(phases[0], cur, stride, self.inner_obj_kind, clip_log_std=clip, grad=g, out_params=nxt,
                           sgd_lr=self.inner_lr, stats=stats_all[0], reuse=self._reuse_bufs)
                chain.append((cur, stride, clip))
                cur, stride, clip = nxt, P, 0
                continue
            g = torch.empty(M, P, dtype=torch.float32, device=dev)
            nxt = torch.empty(M, P, dtype=torch.float32, device=dev)
            self._grad(phases[s], cur, stride, self.inner_obj_kind, clip_log_std=clip, grad=g, out_params=nxt,
                       sgd_lr=self.inner_lr, stats=stats_all[s])
            chain.append((cur, stride, clip))
            cur, stride, clip = nxt, P, 0
        v = torch.empty(M, P, dtype=torch.float32, device=dev) if want_grad else None
        self._grad(phases[-1], cur, stride, outer_obj_kind, obj_scale=outer_obj_scale, clip_eps=clip_eps,
                   kl_coeff=outer_kl_coeff, clip_log_std=clip, grad=v, stats=stats_all[S - 1])
        out = dict(surr=stats_all[S - 1, :, 0], outer_kl=stats_all[S - 1, :, 1], inner_kl=stats_all[:S - 1, :, 1],
                   stats_all=stats_all, grad=None)
        if want_grad:
            for s in range(S - 2, -1, -1):
                prm, strd, clp = chain[s]
                v_out = torch.empty(M, P, dtype=torch.float32, device=dev)
                self._hvp(phases[s], prm, strd, v, v_out, inner_kl_coeffs[s], clp)
                v = v_out
        if explore is not None:
            explore_launch()
            out['explore'] = x_stats[:, 0]
        if want_grad:
            if reduce:
                out['grad'] = reduced(v)
            else:
                out['grad_tasks'] = v
        return out

    def optimize_policy(self, all_samples_data, log=True):
        raise NotImplementedError
