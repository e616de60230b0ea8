"""TRPOMAML (ref: meta_policy_search/meta_algos/trpo_maml.py:8-192) on the GPU."""
import numpy as np

from promp_b200 import _lib
from promp_b200.meta_algos.base import MAMLAlgo
from promp_b200.optimizers.conjugate_gradient_optimizer import ConjugateGradientOptimizer
from promp_b200.utils import logger
from promp_b200.utils.dist import allreduce_sum_, world_size


class TRPOMAML(MAMLAlgo):
    """Same constructor arguments as the reference (trpo_maml.py:23-47)."""

    def __init__(self, *args, name="trpo_maml", step_size=0.01, inner_type='likelihood_ratio', exploration=False,
                 **kwargs):
        if kwargs.get('trainable_inner_step_size', len(args) > 4 and args[4]):
            raise NotImplementedError("TRPOMAML does not support trainable_inner_step_size: the KL trust region has no curvature "
                                      "along the inner step sizes, so conjugate gradient over [theta; alpha] is singular "
                                      "(ProMP and VPGMAML support it)")
        super(TRPOMAML, self).__init__(*args, **kwargs)
        assert inner_type in ["log_likelihood", "likelihood_ratio", "dice"]
        if inner_type == 'dice':
            raise NotImplementedError("inner_type='dice' (reference raises NotImplementedError too, trpo_maml.py:64)")
        self.step_size = step_size
        self.inner_type = inner_type
        self.name = name
        self._optimization_keys = ['observations', 'actions', 'advantages', 'agent_infos']
        self.exploration = exploration
        self.inner_obj_kind = _lib.OBJ_RATIO if inner_type == 'likelihood_ratio' else _lib.OBJ_LOGLIK
        self.optimizer = ConjugateGradientOptimizer()
        self.optimizer.build(self, step_size)

    # ---- E-MAML exploration term (:137-144): surr_i += -mean(adj_avg_rewards_i) * mean(logp_theta(a0 | x0))
    def _exploration_coeff(self, phases):
        """c_i = mean_n adj_avg_rewards_i of the LAST phase = (mean r_i - mean r_all) / (std r_all + 1e-8), on the
        device from the processing kernel's per-task sums (global over ranks), expanded to [M, N].  The eager statement of
        exploration_coeff_dev for fixed-horizon phases, kept as its reference; the algorithms no longer call it."""
        import torch
        last = phases[-1]
        if getattr(last, 'n_valid', None) is not None or getattr(phases[0], 'n_valid', None) is not None:
            raise NotImplementedError("_exploration_coeff covers fixed-horizon paths; exploration_coeff_dev covers both")
        if getattr(last, 'adj_avg_rewards_mean', None) is not None:
            # reference-style sample dicts (MAMLAlgo._phase_of): the caller's processor already computed adj_avg_rewards
            return last.adj_avg_rewards_mean.view(-1, 1).expand(last.M, phases[0].N).contiguous()
        if getattr(last, 'stats', None) is None:
            raise NotImplementedError("exploration=True needs 'adj_avg_rewards' in the sample dicts or a phase processed by "
                                      "promp_b200's MetaSampleProcessor")
        if getattr(last, '_explore_adv', None) is None:
            st = last.stats[:, 5:7]                                    # per task: sum r, sum r^2
            tot = torch.cat([st.sum(0), torch.tensor([float(last.M * last.N)], dtype=torch.float64, device=st.device)])
            allreduce_sum_(tot)
            mean_all = tot[0] / tot[2]
            std_all = torch.sqrt(torch.clamp(tot[1] / tot[2] - mean_all * mean_all, min=0.0))
            c = ((st[:, 0] / last.N - mean_all) / (std_all + 1e-8)).float()
            last._explore_adv = c.view(-1, 1).expand(last.M, phases[0].N).contiguous()
        return last._explore_adv

    def exploration_coeff_dev(self, phases):
        """c [M] float32 on the device: the task means of adj_avg_rewards of the LAST phase, over each task's valid samples
        (promp_emaml_coeff on the processing kernel's per-task reward sums; totals summed over ranks).  No host arithmetic
        and no host copies: a CUDA graph records it.  Computed once per phase and data generation."""
        import torch
        last = phases[-1]
        if getattr(last, 'adj_avg_rewards_mean', None) is not None:
            return last.adj_avg_rewards_mean          # reference-style sample dicts: already the task means
        if getattr(last, 'stats', None) is None:
            raise NotImplementedError("exploration=True needs 'adj_avg_rewards' in the sample dicts or a phase processed by "
                                      "promp_b200's MetaSampleProcessor")
        gen = getattr(last, 'generation', 0)
        cached = getattr(last, '_emaml_coeff', None)
        if cached is not None and cached[0] == gen:
            return cached[1]
        M, dev = last.M, last.stats.device
        n_valid = getattr(last, 'n_valid', None)
        c = torch.empty(M, dtype=torch.float32, device=dev)
        if world_size() > 1:
            tot = torch.empty(3, dtype=torch.float64, device=dev)
            _lib.call('promp_emaml_totals', M, _lib.ptr(last.stats), _lib.ptr(n_valid), last.N, _lib.ptr(tot), _lib.stream())
            allreduce_sum_(tot)
            _lib.call('promp_emaml_finish', M, _lib.ptr(last.stats), _lib.ptr(n_valid), last.N, _lib.ptr(tot), _lib.ptr(c),
                      _lib.stream())
        else:
            _lib.call('promp_emaml_coeff', M, _lib.ptr(last.stats), _lib.ptr(n_valid), last.N, _lib.ptr(c), _lib.stream())
        last._emaml_coeff = (gen, c)
        return c

    def _exploration_term(self, theta, phases, want_grad):
        """(-c_i * mean logp) per task [M] and, optionally, its gradient w.r.t. theta per task [M,P]: one OBJ_EXPLORE
        launch of promp_policy_grad on the phase-0 data.  The meta-objective passes run the same stage inside their chain
        (MAMLAlgo._meta_pass(explore=...)); this stand-alone form serves diagnostics and tests."""
        import torch
        p = self.policy
        st = torch.empty(self.meta_batch_size, 4, dtype=torch.float32, device=p.device)
        g = torch.empty(self.meta_batch_size, p.num_params, dtype=torch.float32, device=p.device) if want_grad else None
        self._grad(phases[0], theta, 0, _lib.OBJ_EXPLORE, clip_log_std=1, grad=g, stats=st, adv=self.exploration_coeff_dev(phases))
        return st[:, 0], g

    def _explore(self, phases):
        return self.exploration_coeff_dev(phases) if self.exploration else None

    # meta objective = mean_i -mean(ratio*adv) (:135,152); constraint = mean_i mean KL(old || theta_i') (:133,149)
    def loss_terms_dev(self, theta, phases, out=None):
        """[loss, inner KLs.., outer KL] at `theta` as a device float32 vector (global means over tasks and ranks), written
        into `out` when given.  No host interaction."""
        import torch
        S1 = self.num_inner_grad_steps
        res = self._meta_pass(theta, phases, _lib.OBJ_RATIO, 0.0, [0.0] * S1, want_grad=False, explore=self._explore(phases))
        if out is None:
            out = torch.empty(S1 + 2, dtype=torch.float32, device=self.policy.device)
        _lib.call('promp_meta_loss_terms', S1 + 1, self.meta_batch_size, _lib.ptr(res['stats_all']),
                  1.0 / (self.meta_batch_size * world_size()), None, S1 + 2, _lib.ptr(out), _lib.stream())
        if self.exploration:
            out[0] += res['explore'].sum() / (self.meta_batch_size * world_size())
        allreduce_sum_(out)
        return out

    def eval_gradient_dev(self, theta, phases, which):
        """Flat gradient [P] of the meta objective ('loss') or of the KL constraint ('kl') at `theta`, all-reduced over
        ranks, on the device."""
        zeros = [0.0] * self.num_inner_grad_steps
        if which == 'loss':
            res = self._meta_pass(theta, phases, _lib.OBJ_RATIO, 0.0, zeros, want_grad=True, explore=self._explore(phases))
        else:
            res = self._meta_pass(theta, phases, _lib.OBJ_NONE, 0.0, zeros, want_grad=True, outer_kl_coeff=1.0)
        allreduce_sum_(res['grad'])
        return res['grad']

    def eval_scalars(self, theta, phases):
        """(loss, mean KL) as host floats (one device->host read; diagnostics / tests)."""
        host = self.loss_terms_dev(theta, phases).cpu().numpy()
        return float(host[0]), float(host[-1])

    def eval_gradient(self, theta, phases, which):
        return self.eval_gradient_dev(theta, phases, which).cpu().numpy().astype(np.float32)

    LOG_KEYS = ('LossBefore', 'MeanKLBefore', 'LossAfter', 'MeanKL', '_accepted_k', '_rejected', '_need_more', '_beta')

    @property
    def graph_capturable(self):
        # Every iteration is device-only, E-MAML included: its coefficient is promp_emaml_coeff (plus an NCCL all-reduce of
        # three float64 totals with several ranks).  The Trainer still runs early-terminating envs eagerly.  (Round 2 ran
        # several ranks eagerly because the ~250-launch capture was invalidated now and then: that was Python's cyclic GC
        # destroying an older CUDAGraph during the capture, fixed in Trainer.capture_graph.)
        return True

    def optimize_phases(self, phases, out=None, want_terms=True):
        """optimize_policy on PhaseData objects up to the verdict on the first line-search group, everything left on the
        device: the CUDA-graph Trainer captures this and reads the float64 result vector back with its logged scalars; if
        the verdict is `need_more` (rare) post_replay() finishes the backtracking eagerly."""
        self._last_phases = phases
        return self.optimizer.optimize_device(phases).double()

    def post_replay(self, hidden, phases):
        """Called by the CUDA-graph Trainer after its one device->host read; `hidden` holds the `_`-prefixed LOG_KEYS."""
        need_more = hidden['_need_more'] != 0.0 if hidden is not None else True     # log=False: the verdict was not read yet
        res = None
        if need_more:
            res = self.optimizer.continue_line_search(phases, self.optimizer._buffers()['result'].cpu().numpy())
        if hidden is not None:
            if res is not None:
                logger.logkv('LossAfter', float(res[2]))
                logger.logkv('MeanKL', float(res[3]))
            kv = logger.getkvs()
            logger.logkv('dLoss', float(kv['LossBefore']) - float(kv['LossAfter']))

    def optimize_policy(self, all_samples_data, log=True):
        """trpo_maml.py:161-192."""
        assert len(all_samples_data) == self.num_inner_grad_steps + 1
        phases = [self._phase_of(s) for s in all_samples_data]
        logger.log("Optimizing")
        res = self.optimizer.optimize(phases)
        loss_before, mean_kl_before, loss_after, mean_kl = (float(v) for v in res[:4])
        self.last_stats = dict(loss_before=loss_before, loss_after=loss_after, kl_before=mean_kl_before, kl=mean_kl)
        if log:
            logger.logkv('MeanKLBefore', mean_kl_before)
            logger.logkv('MeanKL', mean_kl)
            logger.logkv('LossBefore', loss_before)
            logger.logkv('LossAfter', loss_after)
            logger.logkv('dLoss', loss_before - loss_after)
