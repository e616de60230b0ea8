"""MAMLPPOOptimizer (ref: meta_policy_search/optimizers/maml_first_order_optimizer.py:6-163):
`max_epochs` full-batch steps of tf.train.AdamOptimizer on the meta objective with persistent slot
state, then compute_stats.  The Adam update is promp_adam_tf1 (TF1 formula, device step counter).  With trainable inner step
sizes the variables are [theta; alpha] (the reference's var_list with its TODO, meta_algos/base.py:109, done): alpha's Adam
slots live here, one step counter serves both."""
from promp_b200 import _lib
from promp_b200.utils.dist import allreduce_sum_


class MAMLPPOOptimizer(object):
    def __init__(self, learning_rate=1e-3, max_epochs=1, tolerance=1e-6, num_minibatches=1, verbose=False,
                 beta1=0.9, beta2=0.999, epsilon=1e-8):
        self._lr, self._max_epochs = float(learning_rate), int(max_epochs)
        self._tolerance, self._num_minibatches, self._verbose = tolerance, num_minibatches, verbose
        self._b1, self._b2, self._eps = beta1, beta2, epsilon
        self._target = None

    def build(self, policy, alpha=None):
        """build_graph (:48-64): the Adam slots (m, v, step) are created once and persist across iterations.
        alpha: the algorithm's trainable inner step sizes [P] (device), updated together with theta."""
        import torch
        self._target = policy
        P = policy.num_params
        self.m = torch.zeros(P, dtype=torch.float32, device=policy.device)
        self.v = torch.zeros(P, dtype=torch.float32, device=policy.device)
        self.step = torch.zeros(1, dtype=torch.int32, device=policy.device)
        self._ticket = torch.zeros(1, dtype=torch.int32, device=policy.device)      # completion ticket of promp_meta_update
        self.alpha = alpha
        if alpha is None:
            self.m_alpha = self.v_alpha = None
            self.last_grad = torch.zeros(P, dtype=torch.float32, device=policy.device)
        else:
            self.m_alpha = torch.zeros(P, dtype=torch.float32, device=policy.device)
            self.v_alpha = torch.zeros(P, dtype=torch.float32, device=policy.device)
            self.last_grad_full = torch.zeros(2 * P, dtype=torch.float32, device=policy.device)    # [theta; alpha]
            self.last_grad = self.last_grad_full[:P]

    def slots(self):
        """Every tensor of the optimizer's state (the CUDA-graph Trainer saves and restores them around its warm-ups)."""
        return [t for t in (self.m, self.v, self.step, self.m_alpha, self.v_alpha) if t is not None]

    def get_state(self):
        """Adam slots as numpy (snapshots; the reference's tf.train.Saver-less snapshot drops them, we keep them so that a
        resumed run continues bit-identically)."""
        st = dict(m=self.m.cpu().numpy(), v=self.v.cpu().numpy(), step=int(self.step.item()))
        if self.m_alpha is not None:
            st.update(m_alpha=self.m_alpha.cpu().numpy(), v_alpha=self.v_alpha.cpu().numpy())
        return st

    def set_state(self, st):
        import torch
        self.m.copy_(torch.from_numpy(st['m']))
        self.v.copy_(torch.from_numpy(st['v']))
        self.step.fill_(int(st['step']))
        if self.m_alpha is not None and 'm_alpha' in st:
            self.m_alpha.copy_(torch.from_numpy(st['m_alpha']))
            self.v_alpha.copy_(torch.from_numpy(st['v_alpha']))

    def _adam_sgd(self, M, P, scale, task_grads, pairs, grad_in, comm):
        """promp_meta_update_sgd: TF1 Adam over [theta; alpha] (one launch), from per-task gradients or a summed [2P] one."""
        p = self._target
        lam = _lib.ptr_array([a for a, _ in pairs])
        g = _lib.ptr_array([b for _, b in pairs])
        _lib.call('promp_meta_update_sgd', M, P, _lib.ptr(task_grads), len(pairs), lam, g, _lib.ptr(grad_in), scale,
                  _lib.ptr(self.last_grad_full), _lib.ptr(p.theta), _lib.ptr(self.alpha), _lib.ptr(self.m), _lib.ptr(self.v),
                  _lib.ptr(self.m_alpha), _lib.ptr(self.v_alpha), _lib.ptr(self.step), self._lr, self._b1, self._b2, self._eps,
                  *comm, _lib.ptr(self._ticket), _lib.stream())

    def apply_gradient_sgd(self, grad):
        """Adam over [theta; alpha] from the summed [2P] gradient (already all-reduced)."""
        self._adam_sgd(1, self._target.num_params, 1.0, None, [], grad, (1, 0, 0, None, None, None))

    def apply_gradient(self, grad):
        p = self._target
        _lib.call('promp_adam_tf1', p.num_params, _lib.ptr(p.theta), _lib.ptr(grad), _lib.ptr(self.m), _lib.ptr(self.v),
                  _lib.ptr(self.step), self._lr, self._b1, self._b2, self._eps, _lib.stream())

    def apply_task_gradients(self, task_grads):
        """Per-task meta-gradients [M, P] -> task mean -> sum over ranks (NVLink peer memory) -> TF1 Adam, one launch
        (promp_meta_update).  Returns False when the multi-rank case has no peer-memory communicator (NCCL fallback)."""
        from promp_b200.utils import dist as _dist
        p = self._target
        W = _dist.world_size()
        p2p = _dist._p2p
        if W > 1 and (p2p is None or p.num_params > p2p.cap):
            return False
        M = task_grads.shape[0]
        comm = (p2p.world, p2p.rank, p2p.cap, _lib.ptr(p2p.peers), _lib.ptr(p2p.epoch), _lib.ptr(p2p.error)) if W > 1 else \
            (1, 0, 0, None, None, None)
        _lib.call('promp_meta_update', M, p.num_params, _lib.ptr(task_grads), 1.0 / (M * W), _lib.ptr(self.last_grad),
                  _lib.ptr(p.theta), _lib.ptr(self.m), _lib.ptr(self.v), _lib.ptr(self.step), self._lr, self._b1, self._b2,
                  self._eps, *comm, _lib.ptr(self._ticket), _lib.stream())
        return True

    def apply_task_gradients_sgd(self, res):
        """apply_task_gradients over [theta; alpha]: per-task theta gradients and the (v_{s+1}, g_s) pairs -> task mean and
        alpha gradient -> ONE exchange of the 2P values over peer memory -> Adam on both, one launch.  Without a peer-memory
        communicator that holds 2P values: promp_reduce_tasks_sgd, an NCCL all-reduce, then the Adam launch."""
        import torch
        from promp_b200.utils import dist as _dist
        p = self._target
        P, W = p.num_params, _dist.world_size()
        task_grads, pairs = res['grad_tasks'], res['sgd_pairs']
        M = task_grads.shape[0]
        p2p = _dist._p2p
        if W > 1 and (p2p is None or 2 * P > p2p.cap):
            flat = torch.empty(2 * P, dtype=torch.float32, device=p.device)
            lam, g = _lib.ptr_array([a for a, _ in pairs]), _lib.ptr_array([b for _, b in pairs])
            _lib.call('promp_reduce_tasks_sgd', M, P, _lib.ptr(task_grads), len(pairs), lam, g, 1.0 / (M * W), _lib.ptr(flat),
                      _lib.stream())
            allreduce_sum_(flat)
            self.apply_gradient_sgd(flat)
            return
        comm = (p2p.world, p2p.rank, p2p.cap, _lib.ptr(p2p.peers), _lib.ptr(p2p.epoch), _lib.ptr(p2p.error)) if W > 1 else \
            (1, 0, 0, None, None, None)
        self._adam_sgd(M, P, 1.0 / (M * W), task_grads, pairs, None, comm)

    def optimize(self, algo, phases):
        """optimize (:82-115) + compute_stats (:146-163).  Returns a device vector
        [loss_before, loss_after, inner_kl_0.., outer_kl] without synchronising the host."""
        import torch
        S1 = algo.num_inner_grad_steps
        fused = getattr(algo, 'FUSED_LOSS_TERMS', False)
        if fused:
            # [loss_before | loss_after, inner_kls, outer_kl] written in place by promp_meta_loss_terms: no cat / slicing kernels
            final = torch.empty(S1 + 3, dtype=torch.float32, device=algo.policy.device)
        loss_before = None
        fused_update = getattr(algo, 'FUSED_META_UPDATE', False)
        for epoch in range(self._max_epochs):
            res = algo._objective_pass(phases, want_grad=True, reduce=False) if fused_update else \
                algo._objective_pass(phases, want_grad=True)
            if loss_before is None:
                loss_before = algo.loss_terms(res, out=final[0:], n_out=1)[0:1] if fused else algo.loss_terms(res)[0:1]
            if self.alpha is not None:             # [theta; alpha]
                if fused_update:
                    self.apply_task_gradients_sgd(res)
                else:
                    allreduce_sum_(res['grad'])
                    self.apply_gradient_sgd(res['grad'])
                continue
            if fused_update and self.apply_task_gradients(res['grad_tasks']):
                continue                                # task mean + all-reduce + Adam happened in one launch
            if fused_update:                            # no peer-memory communicator: reduce here, all-reduce through NCCL
                flat = torch.empty(algo.policy.num_params, dtype=torch.float32, device=algo.policy.device)
                M = res['grad_tasks'].shape[0]
                from promp_b200.utils.dist import world_size
                _lib.call('promp_reduce_tasks', M, algo.policy.num_params, _lib.ptr(res['grad_tasks']), 1.0 / (M * world_size()),
                          _lib.ptr(flat), _lib.stream())
                res['grad'] = flat
            allreduce_sum_(res['grad'])                 # the ONE collective of the data path: [P] floats over NVLink
            self.apply_gradient(res['grad'])
            self.last_grad = res['grad']
        res = algo._objective_pass(phases, want_grad=False)
        if fused and loss_before is not None:
            algo.loss_terms(res, out=final[1:])
            return final
        terms = algo.loss_terms(res)
        if loss_before is None:
            loss_before = terms[0:1]
        return torch.cat([loss_before, terms])
