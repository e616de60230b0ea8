"""Trainer: the meta-iteration driver.

The reference's own driver (meta_policy_search/meta_trainer.py:7-164) runs UNCHANGED on top of these
classes (see INTEGRATION.md: put promp_b200/tf_shim on sys.path for its `import tensorflow`).  This
module is an independent driver with the same constructor, loop structure and logged keys for use
where the reference tree is absent (the GPU box, bench.py): sample -> process -> adapt, repeated
num_inner_grad_steps times, one more sample/process, then the outer optimisation.
"""
import time

import numpy as np

from promp_b200 import _lib
from promp_b200.utils import logger


def _check_collectives():
    """N > 1: raise if the peer-memory all-reduce timed out on a missing rank (its output is NaN-poisoned from then on)."""
    from promp_b200.utils import dist
    if dist._p2p is not None:
        dist._p2p.check()


class Trainer(object):
    def __init__(self, algo, env, sampler, sample_processor, policy, n_itr, start_itr=0, num_inner_grad_steps=1,
                 sess=None, use_cuda_graph='auto', prefetch_host_inputs=True):
        self.algo, self.env, self.sampler, self.sample_processor = algo, env, sampler, sample_processor
        self.baseline = sample_processor.baseline
        self.policy = policy
        self.n_itr, self.start_itr = n_itr, start_itr
        self.num_inner_grad_steps = num_inner_grad_steps
        self.sess = sess
        # 'auto' (default): train() replays the device part of every iteration as one CUDA graph whenever the configuration
        # allows it (fused fixed-horizon rollouts, ProMP with a fixed KL coefficient), else runs train_iteration eagerly
        self.use_cuda_graph = use_cuda_graph
        self.prefetch_host_inputs = prefetch_host_inputs   # graph mode: draw iteration i+1's host inputs while the GPU runs i
        self._graph_step = None

    def train_iteration(self, itr, log=True):
        t_itr = time.time()
        self.sampler.update_tasks()
        self.policy.switch_to_pre_update()
        all_samples_data = []
        t_sampling = t_proc = t_inner = 0.0
        for step in range(self.num_inner_grad_steps + 1):
            prefix = 'Step_%d-' % step
            t = time.time()
            paths = self.sampler.obtain_samples(log=log, log_prefix=prefix)
            t_sampling += time.time() - t
            t = time.time()
            samples_data = self.sample_processor.process_samples(paths, log='all' if log else False, log_prefix=prefix)
            all_samples_data.append(samples_data)
            t_proc += time.time() - t
            if log:
                self.log_diagnostics(sum(list(paths.values()), []), prefix=prefix)
            t = time.time()
            if step < self.num_inner_grad_steps:
                self.algo._adapt(samples_data)
            t_inner += time.time() - t
        t_outer = time.time()
        self.algo.optimize_policy(all_samples_data, log=log)
        if log:
            _check_collectives()
            logger.logkv('Itr', itr)
            logger.logkv('n_timesteps', self.sampler.total_timesteps_sampled)
            logger.logkv('Time-OuterStep', time.time() - t_outer)
            logger.logkv('Time-MAMLSteps', time.time() - t_outer)
            logger.logkv('Time-TotalInner', t_outer - t_itr)
            logger.logkv('Time-InnerStep', t_inner)
            logger.logkv('Time-SampleProc', t_proc)
            logger.logkv('Time-Sampling', t_sampling)
            logger.logkv('ItrTime', time.time() - t_itr)
        return all_samples_data

    # ------------------------------------------------------------------ CUDA-graph replay of the device part
    def capture_graph(self, warmup=3, log=False, prefetch_host_inputs=False):
        """Capture everything of a meta-iteration that runs on the device (S x [rollout + processing], inner adapt
        steps, K Adam epochs + stats pass: ~40 kernel launches) into ONE CUDA graph and return step().

        step() = host part of the reference iteration (numpy task draw; with reset_mode='numpy' also every phase's
        reset states, in the reference's RNG order) -> H2D into static buffers -> graph replay -> (log=True) one D2H
        copy of the packed vector of logged scalars, emitted under the reference's logger keys.
        prefetch_host_inputs=True (reset_mode='numpy' only) software-pipelines the host half: iteration i+1's numpy draws
        go into a second pinned staging slot while the GPU executes iteration i, so step() only starts the H2D copies and
        the replay.  The draw ORDER is unchanged (same values for the same iteration), but the global numpy RNG is
        consumed one iteration ahead - do not interleave other np.random users with step().
        Requirements: device policy + fixed-horizon device env (ProMP's adaptive KL coefficient rule runs on the device:
        promp_adapt_kl_coeff).  With world_size > 1 the
        NCCL all-reduces of the meta-gradient are captured into the graph as well."""
        import torch
        from promp_b200.samplers.device_data import PhaseData
        sampler, proc, algo, policy = self.sampler, self.sample_processor, self.algo, self.policy
        assert sampler._fused_ok(), "graph mode needs the fused rollout path"
        if getattr(proc.baseline, 'device_kind', None) is None:
            raise ValueError("use_cuda_graph=True needs a device baseline (LinearFeatureBaseline, LinearTimeBaseline, "
                             "ZeroBaseline): %r fits and predicts on the host, which a CUDA graph cannot replay; "
                             "use use_cuda_graph=False or 'auto'" % (proc.baseline,))
        assert hasattr(algo, 'optimize_phases'), "graph mode needs an algorithm with a device-only outer step (ProMP, TRPOMAML)"
        S = self.num_inner_grad_steps + 1
        M, E, H = sampler.meta_batch_size, sampler.envs_per_task, sampler.max_path_length
        numpy_resets = sampler.reset_mode == 'numpy'
        sampler.enable_device_phase_counter()
        inner_env = getattr(self.env, '_wrapped_env', self.env)
        keys = []
        state = {}

        def host_part():
            if numpy_resets:
                return sampler.stage_host_inputs(S)
            sampler.update_tasks()
            return 4 * M * sampler.spec['task_dim']

        def device_part():
            policy.switch_to_pre_update()
            phases = []
            del keys[:]
            logvec = state.get('logvec')          # one float64 device vector holds every logged scalar of the iteration
            off = 0
            for step in range(S):
                phase = PhaseData(M, E, H, sampler.spec['obs_dim'], sampler.spec['act_dim'], sampler.device)
                sampler.rollout_into(phase, sampler._static_init[step] if numpy_resets else None, None)
                proc.process_phase(phase)
                phases.append(phase)
                if log:
                    prefix = 'Step_%d-' % step
                    # six path statistics + AveragePolicyStd in one launch, written in place
                    _lib.call('promp_phase_log_terms', M, phase.act_dim, float(M * E), _lib.ptr(phase.stats), _lib.ptr(phase.log_std),
                              _lib.ptr(logvec[off:off + 7]), _lib.stream())
                    keys.extend(prefix + k for k in proc.PATH_STAT_KEYS)
                    keys.append(prefix + 'AveragePolicyStd')
                    off += 7
                    env_terms = inner_env.device_log_terms(phase)
                    if env_terms is not None:
                        logvec[off:off + env_terms.numel()].copy_(env_terms)
                        keys.extend(prefix + k for k in inner_env.DEVICE_LOG_KEYS)
                        off += env_terms.numel()
                if step < self.num_inner_grad_steps:
                    algo.adapt_phase(phase)
            n_algo = len(algo.LOG_KEYS)
            algo_terms = algo.optimize_phases(phases, out=logvec[off:off + n_algo] if log else None, want_terms=log)
            if log:
                if algo_terms is not None:        # algorithms without an in-place writer return their float64 terms
                    logvec[off:off + n_algo].copy_(algo_terms)
                keys.extend(algo.LOG_KEYS)
                off += n_algo
                state['pinned'][:off].copy_(logvec[:off], non_blocking=True)   # the ONE device->host copy of the iteration
            state['phases'] = phases

        # The warm-up passes below are REAL meta-iterations (they size the allocator pools and JIT nothing, but they do train
        # the policy and consume random numbers).  Everything they touch is saved here and put back after the capture, so
        # that step(0) is the run's first iteration exactly as in eager mode: parameters, Adam slots, the device Philox phase
        # counter, the global numpy stream; with trainable inner step sizes also alpha and its Adam slots.
        opt = getattr(algo, 'optimizer', None)
        alpha = getattr(algo, 'alpha', None)
        torch.cuda.synchronize()
        saved = dict(theta=policy.theta.clone(), alpha=alpha.clone() if alpha is not None else None, np_state=np.random.get_state(),
                     kl_coeff=np.array(algo.inner_kl_coeff, dtype=np.float64) if hasattr(algo, 'inner_kl_coeff') else None,
                     phase_counter_dev=sampler._phase_counter_dev.clone(),
                     adam=[t.clone() for t in opt.slots()] if hasattr(opt, 'slots') else None)
        if log:
            n_env_keys = len(getattr(inner_env, 'DEVICE_LOG_KEYS', ()))
            n_log = S * (7 + n_env_keys) + len(algo.LOG_KEYS)
            state['logvec'] = torch.zeros(n_log, dtype=torch.float64, device=sampler.device)
            state['pinned'] = torch.zeros(n_log, dtype=torch.float64).pin_memory()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                host_part()
                device_part()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        host_part()
        # thread_local: other threads of this process (e.g. the NCCL watchdog polling its events) must not invalidate a long
        # capture (observed with the ~250-launch TRPO-MAML iteration at N = 2)
        # No cyclic garbage collection while the stream is capturing: a collected object that owns CUDA resources (e.g. the
        # CUDAGraph of an earlier Trainer, kept alive by the reference cycle of its step closure) destroys them from this
        # thread, which is a prohibited call during capture and invalidates it (observed: cudaErrorStreamCaptureInvalidated
        # at a random launch of the second Trainer of a process).
        import gc
        gc.collect()
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(graph, capture_error_mode='thread_local'):
                device_part()
        finally:
            if gc_was_enabled:
                gc.enable()
        policy.theta.copy_(saved['theta'])
        if alpha is not None:
            alpha.copy_(saved['alpha'])
        if saved['adam'] is not None:
            for dst, src in zip(opt.slots(), saved['adam']):
                dst.copy_(src)
        sampler._phase_counter_dev.copy_(saved['phase_counter_dev'])
        if saved['kl_coeff'] is not None:
            algo.inner_kl_coeff = saved['kl_coeff']      # the warm-up iterations adapted it (device copy included)
        np.random.set_state(saved['np_state'])
        torch.cuda.synchronize()
        self._graph = graph
        self.graph_d2h_bytes = 8 * len(keys) if log else 0
        n_steps = M * E * H * S

        prefetch = bool(prefetch_host_inputs) and numpy_resets
        state['slot'], state['drawn'] = 0, False

        def step(itr=0, last=False):
            t0 = time.time()
            if prefetch:
                if not state['drawn']:
                    sampler.draw_host_inputs(S, state['slot'])
                self.graph_h2d_bytes = sampler.upload_host_inputs(state['slot'])
            else:
                self.graph_h2d_bytes = host_part()
            graph.replay()
            if prefetch and not last:   # next iteration's host draws overlap the replay that was just enqueued
                state['slot'] ^= 1
                sampler.draw_host_inputs(S, state['slot'])
                state['drawn'] = True
            else:
                state['drawn'] = False   # `last`: the numpy stream ends exactly where the reference's would
            sampler.total_timesteps_sampled += n_steps
            if log:
                torch.cuda.current_stream().synchronize()
                _check_collectives()
                vals = state['pinned'].numpy()
                hidden = {}
                for k, v in zip(keys, vals):
                    if k.startswith('_'):
                        hidden[k] = float(v)          # algorithm-private flags (e.g. TRPO line-search verdict)
                    else:
                        logger.logkv(k, int(v) if k.endswith('NumTrajs') else float(v))
                if hasattr(algo, 'post_replay'):
                    algo.post_replay(hidden, state['phases'])
                if hasattr(algo, 'inner_kl_coeff') and 'KLCoeffInner' not in keys:
                    logger.logkv('KLCoeffInner', float(np.mean(algo.inner_kl_coeff)))
                logger.logkv('Itr', itr)
                logger.logkv('n_timesteps', sampler.total_timesteps_sampled)
                # the reference's per-span timers (meta_trainer.py:131-142) have no meaning inside one graph replay: the
                # columns are kept (progress.csv layout) with the whole replay booked under Time-TotalInner / ItrTime
                dt = time.time() - t0
                for k in ('Time-OuterStep', 'Time-InnerStep', 'Time-SampleProc', 'Time-Sampling', 'Time-MAMLSteps'):
                    logger.logkv(k, float('nan'))
                for s_ in range(S):
                    logger.logkv('Step_%d-PolicyExecTime' % s_, float('nan'))
                    logger.logkv('Step_%d-EnvExecTime' % s_, float('nan'))
                logger.logkv('Time-TotalInner', dt)
                logger.logkv('ItrTime', dt)
            elif hasattr(algo, 'post_replay'):
                algo.post_replay(None, state['phases'])     # e.g. TRPO: read the line-search verdict, finish it if needed
            return state['phases']
        return step

    def graph_capturable(self):
        """True when a meta-iteration has no data-dependent host decision: fused fixed-horizon rollouts, a device baseline
        (not a host baseline object) and an algorithm with a device-only outer step (ProMP - its adaptive inner-KL
        coefficient rule runs on the device - and TRPO-MAML)."""
        return bool(self.sampler._fused_ok() and hasattr(self.algo, 'optimize_phases')
                    and getattr(self.algo, 'graph_capturable', True)
                    and getattr(self.baseline, 'device_kind', None) is not None)

    def train(self):
        """meta_trainer.py:59-152.  The default entry point of a run script."""
        start = time.time()
        use_graph = self.graph_capturable() if self.use_cuda_graph == 'auto' else bool(self.use_cuda_graph)
        for itr in range(self.start_itr, self.n_itr):
            logger.log("\n ---------------- Iteration %d ----------------" % itr)
            if use_graph:
                if self._graph_step is None:
                    self._graph_step = self.capture_graph(log=True, prefetch_host_inputs=self.prefetch_host_inputs)
                self._graph_step(itr, last=(itr == self.n_itr - 1))
            else:
                self.train_iteration(itr)
            logger.logkv('Time', time.time() - start)
            logger.save_itr_params(itr, lambda itr=itr: self.get_itr_snapshot(itr))     # built only when a file is due
            logger.dumpkvs()
        logger.log("Training finished")

    def get_itr_snapshot(self, itr):
        """meta_trainer.py:153-158: {itr, policy, env, baseline} (picklable: the policy pickles its init arguments and a
        host copy of the parameters, policies/base.py:205-215), plus what a bit-identical resume needs and the reference
        drops: optimizer slots, adaptive KL coefficients, the sampled-timesteps counter, trainable inner step sizes."""
        snap = dict(itr=itr, policy=self.policy, env=self.env, baseline=self.baseline)
        extra = dict(total_timesteps_sampled=self.sampler.total_timesteps_sampled)
        opt = getattr(self.algo, 'optimizer', None)
        if hasattr(opt, 'get_state') and getattr(opt, '_target', None) is not None:
            extra['optimizer'] = opt.get_state()
        if hasattr(self.algo, 'inner_kl_coeff'):
            extra['inner_kl_coeff'] = np.asarray(self.algo.inner_kl_coeff, dtype=np.float64).copy()
        if getattr(self.algo, 'alpha', None) is not None:
            extra['alpha'] = self.algo.alpha.cpu().numpy()
        snap['promp_b200_state'] = extra
        return snap

    def restore(self, snapshot):
        """Resume from a snapshot dict or file written by logger.save_itr_params: parameters, optimizer slots, KL
        coefficients and counters are restored into the live objects; training continues at itr + 1."""
        if isinstance(snapshot, str):
            snapshot = logger.load_snapshot(snapshot)
        src = snapshot['policy']
        self.policy.set_params(src.get_param_values() if hasattr(src, 'get_param_values') else src)
        if snapshot.get('baseline') is not None and hasattr(self.baseline, '__setstate__') and hasattr(snapshot['baseline'], '__getstate__'):
            self.baseline.__setstate__(snapshot['baseline'].__getstate__())
        extra = snapshot.get('promp_b200_state', {})
        opt = getattr(self.algo, 'optimizer', None)
        if 'optimizer' in extra and hasattr(opt, 'set_state'):
            opt.set_state(extra['optimizer'])
        if 'alpha' in extra and getattr(self.algo, 'alpha', None) is not None:
            import torch
            self.algo.alpha.copy_(torch.from_numpy(extra['alpha']))
        if 'inner_kl_coeff' in extra and hasattr(self.algo, 'inner_kl_coeff'):
            self.algo.inner_kl_coeff = np.asarray(extra['inner_kl_coeff'], dtype=np.float64).copy()
        self.sampler.total_timesteps_sampled = int(extra.get('total_timesteps_sampled', self.sampler.total_timesteps_sampled))
        self.start_itr = int(snapshot['itr']) + 1
        self._graph_step = None
        return self.start_itr

    def log_diagnostics(self, paths, prefix):
        self.env.log_diagnostics(paths, prefix)
        self.policy.log_diagnostics(paths, prefix)
        self.baseline.log_diagnostics(paths, prefix)
