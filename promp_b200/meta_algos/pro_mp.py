"""ProMP (ref: meta_policy_search/meta_algos/pro_mp.py:9-214) on the GPU."""
import numpy as np

from promp_b200 import _lib
from promp_b200.meta_algos.base import MAMLAlgo
from promp_b200.utils.dist import allreduce_sum_, world_size
from promp_b200.optimizers.maml_first_order_optimizer import MAMLPPOOptimizer
from promp_b200.utils import logger


class ProMP(MAMLAlgo):
    """Same constructor arguments as the reference (pro_mp.py:30-57)."""

    def __init__(self, *args, name="ppo_maml", learning_rate=1e-3, num_ppo_steps=5, num_minibatches=1, clip_eps=0.2,
                 target_inner_step=0.01, init_inner_kl_penalty=1e-2, adaptive_inner_kl_penalty=True,
                 anneal_factor=1.0, **kwargs):
        super(ProMP, self).__init__(*args, **kwargs)
        self.optimizer = MAMLPPOOptimizer(learning_rate=learning_rate, max_epochs=num_ppo_steps,
                                          num_minibatches=num_minibatches)
        self.clip_eps = clip_eps
        self.target_inner_step = target_inner_step
        self.adaptive_inner_kl_penalty = adaptive_inner_kl_penalty
        self._coeff_live = None
        self._inner_kl_coeff = init_inner_kl_penalty * np.ones(self.num_inner_grad_steps)
        self.anneal_coeff = 1
        self.anneal_factor = anneal_factor
        self._optimization_keys = ['observations', 'actions', 'advantages', 'agent_infos']
        self.name = name
        self.kl_coeff = [init_inner_kl_penalty] * self.meta_batch_size * self.num_inner_grad_steps
        self.inner_obj_kind = _lib.OBJ_RATIO                     # _adapt_objective_sym (pro_mp.py:59-65)
        self.optimizer.build(self.policy, alpha=self.alpha)

    FUSED_META_UPDATE = True     # _objective_pass(reduce=False) -> per-task gradients for promp_meta_update

    # ---- inner-KL coefficients: a host array (the reference's attribute) or, while a CUDA-graph Trainer drives the algorithm, a
    # device vector that promp_adapt_kl_coeff updates in place - then an adaptive-KL iteration has no host decision.
    @property
    def inner_kl_coeff(self):
        if self._coeff_live is not None:          # the device copy is the authority: read it back (synchronises)
            self._inner_kl_coeff = self._coeff_live.cpu().numpy().astype(np.float64)
        return self._inner_kl_coeff

    @inner_kl_coeff.setter
    def inner_kl_coeff(self, value):
        self._inner_kl_coeff = np.asarray(value, dtype=np.float64)
        if getattr(self, '_coeff_live', None) is not None:
            import torch
            self._coeff_live.copy_(torch.as_tensor(self._inner_kl_coeff, dtype=torch.float32))

    def _device_coeffs(self):
        """Switch to the device-resident coefficient vector (first call: upload the host values; not inside a capture)."""
        import torch
        if self._coeff_live is None:
            host = np.asarray(self._inner_kl_coeff, dtype=np.float32)
            self._coeff_live = torch.from_numpy(host.copy()).to(self.policy.device)
        return self._coeff_live

    def _objective_pass(self, phases, want_grad, reduce=True):
        """meta_objective = mean_i L_clip,i + mean_s(c_s * mean_i KL_s,i)   (pro_mp.py:151-155)."""
        S1 = max(self.num_inner_grad_steps, 1)
        if self._coeff_live is not None:          # c_s read from the device: the stage gets the 1 / S1 of tf.reduce_mean as its scale
            return self._meta_pass(self.policy.theta, phases, _lib.OBJ_CLIP, self.clip_eps, [1.0 / S1] * self.num_inner_grad_steps,
                                   want_grad, reduce=reduce, inner_kl_coeffs_dev=self._coeff_live)
        coeffs = [float(c) / S1 for c in self._inner_kl_coeff]      # tf.reduce_mean over the S-1 steps
        return self._meta_pass(self.policy.theta, phases, _lib.OBJ_CLIP, self.clip_eps, coeffs, want_grad, reduce=reduce)

    LOG_KEYS = ('LossBefore', 'LossAfter', 'KLInner', 'KLCoeffInner')
    FUSED_LOSS_TERMS = True      # loss_terms(res, out=, n_out=) is one promp_meta_loss_terms launch

    def optimize_phases(self, phases, out=None, want_terms=True):
        """optimize_policy on PhaseData objects, everything left on the device - including the adaptive inner-KL coefficient rule.
        The float64 vector [LossBefore, LossAfter, KLInner, KLCoeffInner] for the CUDA-graph Trainer is written into `out` (one
        tiny launch) when given, else returned."""
        import torch
        if self.adaptive_inner_kl_penalty:
            self._device_coeffs()                # KL coefficients on the device: the adaptive rule below needs no host decision
        stats = self.optimizer.optimize(self, phases)
        self.last_stats_device = stats
        self._last_stats = None
        S1 = self.num_inner_grad_steps
        ret = None
        if out is None and want_terms:
            out = ret = torch.empty(4, dtype=torch.float64, device=stats.device)
        # one tiny launch: the four logged scalars + _adapt_kl_coeff (pro_mp.py:201-214) on the device; out[3] = KLCoeffInner after
        # the update, as the reference logs it
        if want_terms or self.adaptive_inner_kl_penalty:
            coeff = self._coeff_live if self._coeff_live is not None else self._coeff_dev    # fixed: loss_terms' cached device copy
            _lib.call('promp_adapt_kl_coeff', S1, _lib.ptr(stats), float(self.target_inner_step),
                      int(bool(self.adaptive_inner_kl_penalty)), _lib.ptr(coeff) if S1 > 0 else None,
                      _lib.ptr(out) if want_terms else None, _lib.stream())
        return ret

    def optimize_policy(self, all_samples_data, log=True):
        """ProMP.optimize_policy (pro_mp.py:165-199): K Adam epochs on the same data, then a stats pass."""
        import torch
        assert len(all_samples_data) == self.num_inner_grad_steps + 1
        phases = [self._phase_of(s) for s in all_samples_data]
        if log: logger.log("Optimizing")
        stats = self.optimizer.optimize(self, phases)
        self.last_stats_device = stats           # [loss_before, loss_after, inner_kl_0.., outer_kl] on the device
        self._last_stats = None
        if not (log or self.adaptive_inner_kl_penalty):
            return                               # nothing is decided or logged on the host: no synchronisation
        if log: logger.log("Computing statistics")
        ls = self.last_stats                     # one device->host copy for everything logged / decided on the host
        if self.adaptive_inner_kl_penalty:
            if log: logger.log("Updating inner KL loss coefficients")
            self.inner_kl_coeff = self.adapt_kl_coeff(self.inner_kl_coeff, ls['inner_kls'], self.target_inner_step)
        if log:
            logger.logkv('LossBefore', ls['loss_before'])
            logger.logkv('LossAfter', ls['loss_after'])
            logger.logkv('KLInner', np.mean(ls['inner_kls']))
            logger.logkv('KLCoeffInner', np.mean(self.inner_kl_coeff))

    @property
    def last_stats(self):
        if self._last_stats is None:
            host = self.last_stats_device.cpu().numpy().astype(np.float64)
            S1 = self.num_inner_grad_steps
            self._last_stats = dict(loss_before=host[0], loss_after=host[1], inner_kls=host[2:2 + S1],
                                    outer_kl=host[2 + S1])
        return self._last_stats

    def loss_terms(self, res, out=None, n_out=None):
        """Scalar meta objective + KLs (global means) from a _meta_pass result, as a device vector
        [loss, inner_kl_0.., outer_kl] (one promp_meta_loss_terms launch; `out` / `n_out`: write the first n_out values
        into a caller-provided buffer)."""
        import torch
        Mg = self.meta_batch_size * world_size()
        S1 = self.num_inner_grad_steps
        st = res['stats_all']
        if self._coeff_live is not None:
            self._coeff_dev = self._coeff_live                # the live device vector (updated by promp_adapt_kl_coeff)
            self._coeff_key = None
        else:
            key = tuple(float(c) for c in self._inner_kl_coeff)
            if getattr(self, '_coeff_key', None) != key:      # cached on the device (no H2D inside a graph capture)
                self._coeff_dev = torch.tensor(key, dtype=torch.float32, device=st.device)
                self._coeff_key = key
        if out is None:
            out = torch.empty(S1 + 2, dtype=torch.float32, device=st.device)
        n_out = S1 + 2 if n_out is None else n_out
        single = world_size() == 1
        from promp_b200.utils import dist as _dist
        p2p = _dist._p2p
        if not single and p2p is not None:
            # means over all ranks' tasks + KL penalty in ONE launch (peer-memory exchange fused into the terms kernel)
            _lib.call('promp_meta_loss_terms_p2p', S1 + 1, self.meta_batch_size, _lib.ptr(st), 1.0 / Mg,
                      _lib.ptr(self._coeff_dev) if S1 > 0 else None, n_out, _lib.ptr(out), p2p.world, p2p.rank, p2p.cap,
                      _lib.ptr(p2p.peers), _lib.ptr(p2p.epoch), _lib.ptr(p2p.error), _lib.stream())
            return out
        _lib.call('promp_meta_loss_terms', S1 + 1, self.meta_batch_size, _lib.ptr(st), 1.0 / Mg,
                  _lib.ptr(self._coeff_dev) if (single and S1 > 0) else None, n_out if single else S1 + 2, _lib.ptr(out),
                  _lib.stream())
        if not single:                                        # NCCL fallback: sum the per-rank means, then add the penalty
            allreduce_sum_(out)
            if S1 > 0:
                out[0] += (self._coeff_dev * out[1:1 + S1]).mean()
        return out

    def adapt_kl_coeff(self, kl_coeff, kl_values, kl_target):
        """pro_mp.py:201-214."""
        if hasattr(kl_values, '__iter__'):
            assert len(kl_coeff) == len(kl_values)
            return np.array([_adapt_kl_coeff(kl_coeff[i], kl, kl_target) for i, kl in enumerate(kl_values)])
        return _adapt_kl_coeff(kl_coeff, kl_values, kl_target)


def _adapt_kl_coeff(kl_coeff, kl, kl_target):
    if kl < kl_target / 1.5:
        kl_coeff /= 2
    elif kl > kl_target * 1.5:
        kl_coeff *= 2
    return kl_coeff
