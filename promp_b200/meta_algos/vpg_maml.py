"""VPGMAML (ref: meta_policy_search/meta_algos/vpg_maml.py:9-169) on the GPU: vanilla-policy-gradient meta objective
-mean(logp_{theta_i'}(a) * adv) through the inner step(s), one Adam step per meta-iteration
(MAMLFirstOrderOptimizer, max_epochs = 1), optional E-MAML exploration term."""
import numpy as np

from promp_b200 import _lib
from promp_b200.meta_algos.base import MAMLAlgo
from promp_b200.meta_algos.trpo_maml import TRPOMAML
from promp_b200.optimizers.maml_first_order_optimizer import MAMLPPOOptimizer
from promp_b200.utils import logger
from promp_b200.utils.dist import allreduce_sum_, world_size


class VPGMAML(MAMLAlgo):
    """Same constructor arguments as the reference (vpg_maml.py:24-46)."""

    def __init__(self, *args, name="vpg_maml", learning_rate=1e-3, inner_type='likelihood_ratio', exploration=False,
                 **kwargs):
        super(VPGMAML, self).__init__(*args, **kwargs)
        assert inner_type in ["log_likelihood", "likelihood_ratio"]
        self.optimizer = MAMLPPOOptimizer(learning_rate=learning_rate, max_epochs=1)
        self.inner_type = inner_type
        self._optimization_keys = ['observations', 'actions', 'advantages', 'agent_infos']
        self.name = name
        self.exploration = exploration
        if exploration:
            self._optimization_keys.append('adj_avg_rewards')
        self.inner_obj_kind = _lib.OBJ_RATIO if inner_type == 'likelihood_ratio' else _lib.OBJ_LOGLIK
        self.optimizer.build(self.policy, alpha=self.alpha)

    # the E-MAML term is shared with TRPOMAML (same formula, vpg_maml.py:137-144 == trpo_maml.py:137-144).  The Trainer never
    # captures VPGMAML into a CUDA graph (it has no optimize_phases); its coefficient is device-side all the same.
    _exploration_coeff = TRPOMAML._exploration_coeff
    exploration_coeff_dev = TRPOMAML.exploration_coeff_dev
    _exploration_term = TRPOMAML._exploration_term
    _explore = TRPOMAML._explore

    def _objective_pass(self, phases, want_grad):
        zeros = [0.0] * self.num_inner_grad_steps
        res = self._meta_pass(self.policy.theta, phases, _lib.OBJ_LOGLIK, 0.0, zeros, want_grad, explore=self._explore(phases))
        if self.exploration:
            res['surr'] = res['surr'] + res['explore']
        return res

    def loss_terms(self, res):
        import torch
        vec = torch.cat([res['surr'].sum().view(1), res['inner_kl'].sum(1).view(-1), res['outer_kl'].sum().view(1)]) / (
            self.meta_batch_size * world_size())
        return allreduce_sum_(vec)

    def optimize_policy(self, all_samples_data, log=True):
        """vpg_maml.py:147-169: one Adam step, then the loss again."""
        assert len(all_samples_data) == self.num_inner_grad_steps + 1
        phases = [self._phase_of(s) for s in all_samples_data]
        if log: logger.log("Optimizing")
        stats = self.optimizer.optimize(self, phases)
        host = stats.cpu().numpy().astype(np.float64)
        self.last_stats = dict(loss_before=host[0], loss_after=host[1])
        if log:
            logger.logkv('LossBefore', host[0])
            logger.logkv('LossAfter', host[1])
