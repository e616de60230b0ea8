"""MetaSampler on the GPU.

Mirrors meta_policy_search/samplers/meta_sampler.py:12-150 (constructor arguments, attributes,
update_tasks, obtain_samples -> OrderedDict{task: [path]*rollouts}).  With a device policy and a
fixed-horizon device env the whole sampling phase is ONE kernel launch (promp_rollout); otherwise
the reference's step loop runs with the envs stepped on the device (MetaDeviceEnvExecutor).
"""
import time
from collections import OrderedDict

import numpy as np

from promp_b200 import _lib
from promp_b200.samplers.device_data import (PhaseData, LazyPath, LazyPathList, PathsMetaBatch, DeviceRaggedPhaseData,
                                              RaggedLazyPathList)
from promp_b200.samplers.vectorized_env_executor import MetaDeviceEnvExecutor
from promp_b200.utils import dist, logger
from promp_b200.utils.dist import shard_tasks


class MetaSampler(object):
    """
    Args (as the reference):
        env, policy, rollouts_per_meta_task, meta_batch_size, max_path_length, envs_per_task, parallel
    Extra keyword arguments (device specific, all optional):
        reset_mode ('numpy'|'device'): 'numpy' draws task / reset states from the global numpy RNG in the
            reference's consumption order and uploads them (seed-for-seed parity); 'device' draws reset
            states in-kernel with Philox (nothing crosses PCIe).
        seed (int): Philox key for in-kernel action noise / reset states.
        task_shard ((rank, world)): this process owns tasks [rank*M, (rank+1)*M) of a global batch of
            world*M tasks; every rank draws the same global task list and keeps its slice.  On the fused paths a
            sharded run samples exactly what one process with the global batch samples for the same seeds: the rollout
            kernels key their Philox streams by the global env index (task offset rank*M), reset_mode='numpy' draws
            the global batch's reset states and keeps this rank's rows, and early-terminating envs (reset_mode='device')
            cut their timelines where the completed paths of ALL ranks' tasks reach world*M*E*H samples (the per-step
            histogram is summed over ranks with utils.dist.allreduce_sum_).  Not covered: the step loop over
            promp_env_step (early-terminating envs with reset_mode='numpy') and duck-typed host envs reset envs one at
            a time from the host stream, so their reset draws stay per rank.
    `parallel` is accepted and ignored: there are no env worker processes on the device path.
    """

    def __init__(self, env, policy, rollouts_per_meta_task, meta_batch_size, max_path_length, envs_per_task=None,
                 parallel=False, reset_mode='numpy', seed=0, task_shard=None):
        assert hasattr(env, 'reset') and hasattr(env, 'step')
        assert hasattr(env, 'set_task')
        assert reset_mode in ('numpy', 'device')
        self.env, self.policy = env, policy
        self.batch_size = rollouts_per_meta_task
        self.max_path_length = max_path_length
        self.envs_per_task = rollouts_per_meta_task if envs_per_task is None else envs_per_task
        self.meta_batch_size = meta_batch_size
        self.total_samples = meta_batch_size * rollouts_per_meta_task * max_path_length
        self.parallel = parallel
        self.total_timesteps_sampled = 0
        self.reset_mode = reset_mode
        self.seed = int(seed)
        self.task_shard = task_shard
        # world > 1: global index of this rank's first task (Philox key offset) and the number of ranks
        self._shard_world = int(task_shard[1]) if task_shard is not None else 1
        self._task_offset = int(task_shard[0]) * meta_batch_size if self._shard_world > 1 else 0
        self._phase_counter = 0
        self._phase_counter_dev = None      # device uint64 phase counter (graph mode)
        self._injected_noise = None
        self._injected_init = None
        if hasattr(env, 'device_spec'):
            self.vec_env = MetaDeviceEnvExecutor(env, self.meta_batch_size, self.envs_per_task, self.max_path_length)
            self.spec = self.vec_env.spec
            self.device = self.vec_env.device
            if self.spec.get('module') is not None and hasattr(policy, 'hidden_arg'):
                self.spec['module'].handle(policy.hidden_arg)     # a user env: its rollout kernels, loaded before any capture
        else:
            # duck-typed host env (the reference's test fakes, tests/test_samplers.py:13-67): stepped where Python runs,
            # one env.step per env per step like the reference's iterative executor - slow by construction
            from promp_b200.samplers.host_env_executor import MetaHostEnvExecutor
            self.vec_env = MetaHostEnvExecutor(env, self.meta_batch_size, self.envs_per_task, self.max_path_length)
            self.spec, self.device = None, None

    # ------------------------------------------------------------------------------------------
    def update_tasks(self):
        """meta_sampler.py:51-57."""
        tasks = self._draw_tasks()
        assert len(tasks) == self.meta_batch_size
        self.vec_env.set_tasks(tasks)

    def inject(self, noise=None, init_state=None):
        """Parity hooks: action noise [M,E,H,Da] and/or reset states [M,E,state_dim] for the NEXT phase."""
        self._injected_noise, self._injected_init = noise, init_state

    def _fused_ok(self):
        return (self.spec is not None and hasattr(self.policy, 'sampling_params')
                and not self.spec['ends_early'] and self.envs_per_task == self.batch_size)

    def _fused_early_ok(self):
        """Early-terminating envs (MetaPointEnv, the Walker2d surrogates) through the fused kernel + device-side path table.
        Opt-in via reset_mode='device': in-kernel resets cannot follow the host numpy stream (their number is data-dependent),
        so reset_mode='numpy' keeps the reference's step loop with host draws."""
        return (self.spec is not None and hasattr(self.policy, 'sampling_params')
                and self.spec['ends_early']
                and self.reset_mode == 'device' and self.envs_per_task == self.batch_size and self.envs_per_task <= 1024)

    def obtain_samples(self, log=False, log_prefix=''):
        """meta_sampler.py:59-137."""
        t0 = time.time()
        if self._fused_ok():
            paths = self._obtain_samples_fused()
            policy_time, env_time = 0.0, time.time() - t0      # one fused kernel: not separable
        elif self._fused_early_ok():
            paths = self._obtain_samples_fused_early()
            policy_time, env_time = 0.0, time.time() - t0
        else:
            paths, policy_time, env_time = self._obtain_samples_stepwise()
        self.total_timesteps_sampled += self.total_samples
        if log:
            logger.logkv(log_prefix + "PolicyExecTime", policy_time)
            logger.logkv(log_prefix + "EnvExecTime", env_time)
        return paths

    # ------------------------------------------------------------------------------------------
    def rollout_into(self, phase, init_state=None, noise=None):
        """Launch the fused rollout kernel for one sampling phase into `phase` (device buffers)."""
        import torch
        s = self.spec
        M, E, H = self.meta_batch_size, self.envs_per_task, self.max_path_length
        params, stride, clip = self.policy.sampling_params()
        if s['ninfo'] and phase.info is None:
            keys = tuple(getattr(getattr(self.env, '_wrapped_env', self.env), 'info_keys', ('reward_run', 'reward_ctrl')))
            phase.info = torch.empty(len(keys), M, E * H, dtype=torch.float32, device=self.device)
            phase.info_keys = keys
        self._phase_counter += 1
        args = (s['env_kind'], s['reward_type'], s['radius'], int(s.get('normalized', False)), M, E, H, self.policy.hidden_arg,
                _lib.ptr(params), stride, _lib.ptr(self.vec_env.task_params_per_task), _lib.ptr(init_state),
                _lib.ptr(noise), self.seed, self._phase_counter, _lib.ptr(self._phase_counter_dev), clip,
                float(self.policy.min_log_std),
                _lib.ptr(phase.obs), _lib.ptr(phase.act), _lib.ptr(phase.mean), _lib.ptr(phase.rew),
                _lib.ptr(phase.done), _lib.ptr(phase.info), _lib.ptr(phase.log_std), None, _lib.stream())
        if s.get('module') is not None:
            _lib.call('promp_rollout_module', s['module'].handle(self.policy.hidden_arg), *args[1:], self._task_offset)
        elif self._shard_world > 1:
            _lib.call('promp_rollout_ex', *args, self._task_offset)
        else:
            _lib.call('promp_rollout', *args)
        if self._phase_counter_dev is not None:
            _lib.call('promp_counter_add', _lib.ptr(self._phase_counter_dev), 1 << 20, _lib.stream())
        phase.invalidate_host()
        return phase

    def _draw_tasks(self):
        """The reference's task draw (meta_sampler.py:51-57) for this rank's shard; host objects only."""
        if self.task_shard is None:
            return self.env.sample_tasks(self.meta_batch_size)
        rank, world = self.task_shard
        return shard_tasks(self.env.sample_tasks(self.meta_batch_size * world), rank, world)

    def _host_reset_states(self, inner, n):
        """n = M*E reset states from the global numpy RNG for this rank: a sharded run draws the global batch's
        world*M*E states (the draws are vectorised per coordinate block, so a local draw is not a slice of the global
        one) and keeps its rows, so that the values and the stream position match a one-process run."""
        if self._shard_world == 1:
            return inner.host_reset_states(n)
        r0 = self.task_shard[0] * n
        return inner.host_reset_states(self._shard_world * n)[r0:r0 + n]

    def draw_host_inputs(self, n_phases, slot=0):
        """Graph mode with reset_mode='numpy', host half: draw one iteration's tasks and every phase's reset states from
        the global numpy RNG in the reference's consumption order (sample_tasks; then per phase: M*E resets, and the M*E
        end-of-horizon resets whose observations the reference discards) into PINNED staging buffers (two slots, so the
        next iteration can be drawn while the previous upload may still be in flight).  No device interaction."""
        import torch
        M, E = self.meta_batch_size, self.envs_per_task
        inner = getattr(self.env, '_wrapped_env', self.env)
        sd, td = self.spec['state_dim'], self.spec['task_dim']
        if getattr(self, '_pinned_init', None) is None or len(self._pinned_init[0]) != n_phases:
            # ONE device buffer / ONE pinned buffer per slot hold [tasks | reset states of every phase]: a single H2D copy per
            # iteration; the rollout kernels read views of the device buffer (stable addresses: CUDA-graph safe)
            n_task, n_init = (M * td + 3) // 4 * 4, (M * E * sd + 3) // 4 * 4       # 16-byte aligned sections
            self._static_all = torch.empty(n_task + n_phases * n_init, dtype=torch.float32, device=self.device)
            self._pinned_all = [torch.empty(n_task + n_phases * n_init, dtype=torch.float32).pin_memory() for _ in range(2)]
            self._static_init = [self._static_all[n_task + s * n_init:n_task + s * n_init + M * E * sd].view(M, E, sd) for s in range(n_phases)]
            self._pinned_init = [[pa[n_task + s * n_init:n_task + s * n_init + M * E * sd].view(M, E, sd) for s in range(n_phases)]
                                 for pa in self._pinned_all]
            self._pinned_tasks = [pa[:M * td].view(M, td) for pa in self._pinned_all]
            self.vec_env.task_params_per_task = self._static_all[:M * td].view(M, td)
            self._staged_tasks = [None, None]
            self._upload_done = [None, None]
        if self._upload_done[slot] is not None:
            # the H2D copies issued from this pinned slot may still be queued behind an unfinished replay: the host must
            # not overwrite the staging memory before they have executed (it would tear tasks / reset states)
            self._upload_done[slot].synchronize()
        tasks = self._draw_tasks()
        assert len(tasks) == self.meta_batch_size
        self._staged_tasks[slot] = list(tasks)
        self._pinned_tasks[slot].copy_(torch.from_numpy(np.stack([inner.task_vector(t) for t in tasks]).astype(np.float32)))
        for s in range(n_phases):
            self._pinned_init[slot][s].copy_(torch.from_numpy(self._host_reset_states(inner, M * E).astype(np.float32)
                                                              .reshape(M, E, sd)))
            self._host_reset_states(inner, M * E)     # discarded end-of-horizon resets (vectorized_env_executor.py:47-50)

    def upload_host_inputs(self, slot=0):
        """Device half: start the H2D copies of a drawn slot into the static buffers the captured rollouts read."""
        ve = self.vec_env
        ve.tasks = self._staged_tasks[slot]
        if len(ve.tasks):
            self.env.set_task(ve.tasks[-1])
        self._static_all.copy_(self._pinned_all[slot], non_blocking=True)      # tasks + all reset states: one H2D copy
        ve._per_env_tasks_stale = True      # the per-env expansion (stepwise path only) is rebuilt on demand
        import torch
        if self._upload_done[slot] is None:
            self._upload_done[slot] = torch.cuda.Event()
        self._upload_done[slot].record()       # draw_host_inputs(slot) waits on this before reusing the pinned buffers
        M, E = self.meta_batch_size, self.envs_per_task
        n_phases = len(self._static_init)
        return 4 * (M * self.spec['task_dim'] + n_phases * M * E * self.spec['state_dim'])

    def stage_host_inputs(self, n_phases):
        """draw_host_inputs + upload_host_inputs for the current iteration (no look-ahead)."""
        self.draw_host_inputs(n_phases, 0)
        return self.upload_host_inputs(0)

    def enable_device_phase_counter(self):
        """Keep the Philox phase counter in device memory so that a captured CUDA graph draws fresh
        noise / reset states on every replay."""
        import torch
        if self._phase_counter_dev is None:
            self._phase_counter_dev = torch.zeros(1, dtype=torch.int64, device=self.device)

    def _obtain_samples_fused(self):
        import torch
        M, E, H = self.meta_batch_size, self.envs_per_task, self.max_path_length
        inner = getattr(self.env, '_wrapped_env', self.env)
        init = self._injected_init
        if init is None and self.reset_mode == 'numpy':
            # vec_env.reset(): M*E reset draws in env order (vectorized_env_executor.py:73)
            init = self._host_reset_states(inner, M * E).astype(np.float32)
        if init is not None and not isinstance(init, torch.Tensor):
            init = torch.from_numpy(np.ascontiguousarray(init, dtype=np.float32).reshape(M, E, -1)).to(self.device, non_blocking=True)
        noise = self._injected_noise
        if noise is not None and not isinstance(noise, torch.Tensor):
            noise = torch.from_numpy(np.ascontiguousarray(noise, dtype=np.float32)).to(self.device)
        phase = PhaseData(M, E, H, self.spec['obs_dim'], self.spec['act_dim'], self.device)
        self.rollout_into(phase, init, noise)
        if self._injected_init is None and self.reset_mode == 'numpy':
            # at ts == H every env is reset once more and that observation is discarded
            # (vectorized_env_executor.py:47-50): consume the same draws to stay aligned with the reference
            self._host_reset_states(inner, M * E)
        self._injected_noise = self._injected_init = None
        paths = PathsMetaBatch()
        cache = {}
        for m in range(M):
            paths[m] = LazyPathList(phase, (m,), cache)
        paths.phase = phase
        return paths

    def _obtain_samples_fused_early(self):
        """Early-terminating env, no host round trip per step: promp_rollout_early_term records a timeline of 2H-1 steps per
        env slot (paths end on done / horizon, slots reset in-kernel), promp_paths_finalize applies the reference's
        collect-until-M*E*H-samples rule and path ordering on the device and compacts the kept paths into the ragged layout
        the processing / policy kernels take."""
        import torch
        s = self.spec
        M, E, H = self.meta_batch_size, self.envs_per_task, self.max_path_length
        T = 2 * H - 1
        Do, Da, dev = s['obs_dim'], s['act_dim'], self.device
        f32 = dict(dtype=torch.float32, device=dev)
        tl = getattr(self, '_timeline', None)
        if tl is None:
            tl = self._timeline = dict(obs=torch.empty(M, E, T, Do, **f32), act=torch.empty(M, E, T, Da, **f32),
                                       mean=torch.empty(M, E, T, Da, **f32), rew=torch.empty(M, E, T, **f32),
                                       done=torch.empty(M, E, T, dtype=torch.uint8, device=dev),
                                       ws=torch.zeros(_lib.load().promp_paths_workspace_bytes(M, E, T) // 4 + 2, dtype=torch.int32, device=dev))
        n_alloc = (E * T + 3) // 4 * 4        # row stride of the ragged tensors (the policy kernels want a multiple of 4)
        phase = DeviceRaggedPhaseData(M, E * T, n_alloc, Do, Da, dev)
        params, stride, clip = self.policy.sampling_params()
        noise = self._injected_noise
        if noise is not None and not isinstance(noise, torch.Tensor):
            noise = torch.from_numpy(np.ascontiguousarray(noise, dtype=np.float32)).to(dev)
        init = self._injected_init
        if init is not None and not isinstance(init, torch.Tensor):
            init = torch.from_numpy(np.ascontiguousarray(init, dtype=np.float32).reshape(M, E, -1)).to(dev)
        self._injected_noise = self._injected_init = None
        self._phase_counter += 1
        args = (s['env_kind'], int(s.get('normalized', False)), M, E, T, H, self.policy.hidden_arg,
                _lib.ptr(params), stride, _lib.ptr(self.vec_env.task_params_per_task), _lib.ptr(init), _lib.ptr(noise), self.seed,
                self._phase_counter, _lib.ptr(self._phase_counter_dev), clip, float(self.policy.min_log_std), _lib.ptr(tl['obs']),
                _lib.ptr(tl['act']), _lib.ptr(tl['mean']), _lib.ptr(tl['rew']), _lib.ptr(tl['done']), _lib.ptr(phase.log_std),
                _lib.stream())
        if s.get('module') is not None:
            _lib.call('promp_rollout_early_term_module', s['module'].handle(self.policy.hidden_arg), *args[1:], self._task_offset)
        elif self._shard_world > 1:
            _lib.call('promp_rollout_early_term_ex', *args, self._task_offset)
        else:
            _lib.call('promp_rollout_early_term', *args)
        head = (M, E, T, E * T, n_alloc, Do, Da)
        tail = (_lib.ptr(tl['done']), _lib.ptr(tl['obs']), _lib.ptr(tl['act']), _lib.ptr(tl['mean']), _lib.ptr(tl['rew']),
                _lib.ptr(phase.path_off), _lib.ptr(phase.n_paths), _lib.ptr(phase.n_valid), _lib.ptr(phase.src_slot),
                _lib.ptr(phase.src_start), _lib.ptr(phase.obs), _lib.ptr(phase.act), _lib.ptr(phase.mean), _lib.ptr(phase.rew),
                _lib.ptr(phase.done), _lib.ptr(phase.cut), _lib.ptr(tl['ws']), tl['ws'].numel() * 4, _lib.stream())
        if self._shard_world > 1:
            # the reference's rule over the WHOLE task batch (meta_sampler.py:87-137): t* is the first step at which the
            # completed paths of every rank's tasks hold world*M*E*H samples, so the per-step counts are summed over ranks
            # (int32: NCCL) before the cut
            hist = getattr(self, '_shard_hist', None)
            if hist is None:
                hist = self._shard_hist = torch.empty(T, dtype=torch.int32, device=dev)
            hist.zero_()
            _lib.call('promp_paths_histogram', M, E, T, _lib.ptr(tl['done']), _lib.ptr(hist), _lib.stream())
            dist.allreduce_sum_(hist)
            _lib.call('promp_paths_finalize_ex', *head, self._shard_world * M * E * H, _lib.ptr(hist), *tail)
        else:
            _lib.call('promp_paths_finalize', *head, M * E * H, *tail)
        phase.timeline = tl                 # kept for diagnostics / tests (overwritten by the next phase)
        phase.invalidate_host()
        paths = PathsMetaBatch()
        for m in range(M):
            paths[m] = RaggedLazyPathList(phase, m)
        paths.phase = phase
        return paths

    # ------------------------------------------------------------------------------------------
    def _obtain_samples_stepwise(self):
        """The reference loop (meta_sampler.py:76-131), envs stepped by promp_env_step."""
        paths = OrderedDict((i, []) for i in range(self.meta_batch_size))
        n_envs = self.vec_env.num_envs
        running = [dict(observations=[], actions=[], rewards=[], env_infos=[], agent_infos=[]) for _ in range(n_envs)]
        n_samples, policy_time, env_time = 0, 0.0, 0.0
        obses = self.vec_env.reset()
        while n_samples < self.total_samples:
            t = time.time()
            obs_per_task = np.split(np.asarray(obses), self.meta_batch_size)
            actions, agent_infos = self.policy.get_actions(obs_per_task)
            policy_time += time.time() - t
            t = time.time()
            actions = np.concatenate(actions)
            next_obses, rewards, dones, env_infos = self.vec_env.step(actions)
            env_time += time.time() - t
            if not env_infos:
                env_infos = [dict() for _ in range(n_envs)]
            if not agent_infos:
                agent_infos = [dict() for _ in range(n_envs)]
            else:
                assert len(agent_infos) == self.meta_batch_size
                agent_infos = sum(agent_infos, [])
            for idx in range(n_envs):
                r = running[idx]
                r["observations"].append(obses[idx])
                r["actions"].append(actions[idx])
                r["rewards"].append(rewards[idx])
                r["env_infos"].append(env_infos[idx])
                r["agent_infos"].append(agent_infos[idx])
                if dones[idx]:
                    paths[idx // self.envs_per_task].append(dict(
                        observations=np.asarray(r["observations"]), actions=np.asarray(r["actions"]),
                        rewards=np.asarray(r["rewards"]), env_infos=_stack(r["env_infos"]),
                        agent_infos=_stack(r["agent_infos"])))
                    n_samples += len(r["rewards"])
                    running[idx] = dict(observations=[], actions=[], rewards=[], env_infos=[], agent_infos=[])
            obses = next_obses
        return paths, policy_time, env_time


def _stack(dict_list):
    if not dict_list or not dict_list[0]:
        return {}
    return {k: (_stack([d[k] for d in dict_list]) if isinstance(dict_list[0][k], dict)
                else np.asarray([d[k] for d in dict_list])) for k in dict_list[0]}
