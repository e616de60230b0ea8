"""A run sharded over W ranks (MetaSampler(task_shard=(rank, W))) samples exactly what one process samples for the same
global task batch and seeds.

The shards are emulated one after another on one GPU: every shard starts from the same numpy seed and Philox seed as the
global run, and each shard's phase must equal its rows [rank*M, (rank+1)*M) of the global phase bit for bit.
  * fixed horizons (promp_rollout_ex), reset_mode 'numpy' (the global batch's reset draws, this rank's rows) and 'device'
    (Philox keyed by the global env index), two iterations of two phases: the numpy stream stays aligned;
  * early termination (promp_rollout_early_term_ex + promp_paths_histogram + promp_paths_finalize_ex): the timelines, the
    summed histograms, and the path table cut where the completed paths of the WHOLE batch reach W*M*E*H samples - the
    sampler's exchange (utils.dist.allreduce_sum_) is monkeypatched to hand back the global histogram;
  * the C ABI: offset 0 is the base entry point bit for bit, finalize_ex with the local histogram is promp_paths_finalize,
    bad arguments are rejected;
  * on two GPUs (skipped with fewer): Trainer.train() with ProMP at world 2 against one process with the global batch.

Run as a script under torch.distributed.run, this file is the two-GPU worker."""
import os
import signal
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NP_SEED, PHILOX_SEED = 11, 7
FIXED_ENVS = ('point_corner', 'cheetah', 'swimmer')
EARLY_ENVS = ('point', 'walker_vel', 'walker_direc')
ERR = -1        # PROMP_ERR_INVALID_ARG


def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _make_env(name):
    from promp_b200 import envs
    cls = dict(point_corner=envs.MetaPointEnvCorner, cheetah=envs.HalfCheetahRandDirecEnv, swimmer=envs.SwimmerRandVelEnv,
               point=envs.MetaPointEnv, walker_vel=envs.Walker2DRandVelEnv, walker_direc=envs.Walker2DRandDirecEnv)[name]
    return envs.normalize(cls())


def _point_theta(policy, gain):
    """theta of a policy with mean ~= -100 * gain * obs and sigma = e^-10 on normalize(MetaPointEnv) (a_env = clip(0.01 a,
    +-0.1)): at gain 1 the point walks 0.1 per step to the origin and its paths end within ~30 steps; at a small gain it
    creeps and most paths run to the horizon."""
    from oracle import tf_cases
    par = tf_cases.unflatten(np.zeros(policy.num_params_logical, np.float32), 2, 2, 64)
    c = 0.01
    par['mean_network/hidden_0/kernel'][0, 0] = par['mean_network/hidden_0/kernel'][1, 1] = c
    par['mean_network/hidden_1/kernel'][0, 0] = par['mean_network/hidden_1/kernel'][1, 1] = 1.0
    par['mean_network/output/kernel'][0, 0] = par['mean_network/output/kernel'][1, 1] = -100.0 * gain / c
    par['log_std_network/log_std_var'][:] = -10.0
    policy.set_params(par)
    return policy.theta.clone()


def _policy(torch, name, env, M):
    """The policy of a case; its parameters do not depend on M (pre-update: one shared parameter vector)."""
    from promp_b200.policies import MetaGaussianMLPPolicy
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=env.obs_dim, action_dim=env.act_dim, meta_batch_size=M, hidden_sizes=(64, 64))
    if name == 'point':
        _point_theta(policy, 1.0)
    elif name.startswith('walker'):
        from oracle import locomotion_surrogates as ls
        theta = policy.theta.cpu().numpy().copy()
        theta[-6:] = np.log(10.0)                                 # a falling walker: paths of every length
        theta[-12:-6] = 2.0 * np.sign(ls.Walker.P)
        policy.set_params(theta)
    return policy


def _task_thetas(torch, name, policy, MG):
    """Per-task parameters [MG, P] for a post-update early-termination phase (seeded, independent of the shard).  The
    first half of the tasks ends its paths sooner than the second half, so a shard's own first crossing of M*E*H lies at
    another step than the batch's."""
    if name == 'point':
        slow, fast = _point_theta(policy, 0.05), _point_theta(policy, 1.0)
        return torch.stack([fast if m < MG // 2 else slow for m in range(MG)])
    theta = policy.theta.clone()
    rng = np.random.RandomState(5)
    out = theta.unsqueeze(0).repeat(MG, 1)
    out += 0.05 * torch.from_numpy(rng.randn(*out.shape).astype(np.float32)).cuda()
    out[:, -6:] = torch.tensor([np.log(10.0) if m < MG // 2 else np.log(0.5) for m in range(MG)], device='cuda').unsqueeze(1)
    return out


def _sampler(torch, name, M, E, H, reset_mode, shard):
    """(env, policy, sampler) for M local tasks, built from NP_SEED; the numpy stream is re-seeded last, so the global run
    and every shard draw their tasks and reset states from the same stream position."""
    from promp_b200.samplers import MetaSampler
    np.random.seed(NP_SEED)
    env = _make_env(name)
    policy = _policy(torch, name, env, M)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          reset_mode=reset_mode, seed=PHILOX_SEED, task_shard=shard)
    np.random.seed(NP_SEED + 1)
    return env, policy, sampler


def _fixed_phase(ph):
    return {k: getattr(ph, k).cpu().numpy() for k in ('obs', 'act', 'mean', 'rew', 'done')}


def _ragged_phase(ph):
    out = {k: getattr(ph, k).cpu().numpy() for k in ('cut', 'n_paths', 'n_valid', 'path_off', 'src_slot', 'src_start',
                                                     'obs', 'act', 'mean', 'rew', 'done')}
    out.update({'tl_' + k: v.cpu().numpy() for k, v in ph.timeline.items() if k in ('obs', 'act', 'mean', 'rew', 'done')})
    return out


def _assert_fixed_slice(glob, shard, r, M, what):
    for k, v in shard.items():
        assert np.array_equal(_bits(v), _bits(glob[k][r * M:(r + 1) * M])), (what, k)


def _assert_ragged_slice(glob, shard, r, M, what):
    """Cut, path table, compacted rows (up to n_valid) and timelines of shard r equal rows [r*M, (r+1)*M) of the global
    phase, bit for bit."""
    sl = slice(r * M, (r + 1) * M)
    assert list(shard['cut']) == list(glob['cut']), (what, 'cut', list(shard['cut']), list(glob['cut']))
    for k in ('n_paths', 'n_valid', 'path_off'):
        np.testing.assert_array_equal(shard[k], glob[k][sl], err_msg='%s %s' % (what, k))
    for m in range(M):
        n, nv = int(shard['n_paths'][m]), int(shard['n_valid'][m])
        for k in ('src_slot', 'src_start'):
            np.testing.assert_array_equal(shard[k][m, :n], glob[k][r * M + m, :n], err_msg='%s %s %d' % (what, k, m))
        for k in ('obs', 'act', 'mean', 'rew', 'done'):
            assert np.array_equal(_bits(shard[k][m, :nv]), _bits(glob[k][r * M + m, :nv])), (what, k, m)
    for k in ('tl_obs', 'tl_act', 'tl_mean', 'tl_rew', 'tl_done'):
        assert np.array_equal(_bits(shard[k]), _bits(glob[k][sl])), (what, k)


# ================================================================================================================ CPU
def test_ex_entry_points_reject_bad_arguments():
    """A negative task offset, a global env index past the 32-bit Philox key, and bad promp_paths_histogram arguments are
    rejected before anything is launched (the pointers are dummy addresses that must never be dereferenced)."""
    from promp_b200 import _lib
    lib = _lib.load()
    x = 16

    def rollout(M, E, off):
        return lib.promp_rollout_ex(_lib.ENV_POINT_CORNER, _lib.REWARD_DENSE, 0.5, 1, M, E, 10, 64, x, 0, x, None, None, 0, 0, None,
                                    0, 0.0, x, x, x, x, x, None, x, None, None, off)

    def early(M, E, off):
        return lib.promp_rollout_early_term_ex(_lib.ENV_POINT, 1, M, E, 19, 10, 64, x, 0, x, None, None, 0, 0, None, 0, 0.0, x, x,
                                               x, x, x, x, None, off)

    for fn, name in ((rollout, 'promp_rollout_ex'), (early, 'promp_rollout_early_term_ex')):
        for M, E, off, msg in ((2, 5, -1, 'task_offset must be >= 0'), (2, 5, -(1 << 31), 'task_offset must be >= 0'),
                               (1, 1 << 16, (1 << 16), 'exceeds the 32-bit Philox env key'),
                               (4, 1 << 20, (1 << 12) - 3, 'exceeds the 32-bit Philox env key'),
                               (1, 1024, (1 << 31) - 1, 'exceeds the 32-bit Philox env key')):
            assert fn(M, E, off) == ERR, (name, M, E, off)
            err = _lib.last_error()
            assert err.startswith(name + ':') and msg in err, (name, err)
    for args, msg in (((0, 4, 9, x, x), 'sizes must be positive'), ((2, 0, 9, x, x), 'sizes must be positive'),
                      ((2, 4, 0, x, x), 'sizes must be positive'), ((2, -4, 9, x, x), 'sizes must be positive'),
                      ((1 << 16, 1 << 16, 9, x, x), 'exceeds the int32 range'),
                      ((2, 4, 9, None, x), 'null pointer'), ((2, 4, 9, x, None), 'null pointer')):
        assert lib.promp_paths_histogram(*args, None) == ERR, args
        assert msg in _lib.last_error(), (args, _lib.last_error())


def test_finalize_ex_argument_checks():
    """promp_paths_finalize_ex checks what promp_paths_finalize checks, under its own name."""
    from promp_b200 import _lib
    lib = _lib.load()
    x, M, E, T = 16, 2, 4, 9
    ws = lib.promp_paths_workspace_bytes(M, E, T)
    for kw, msg in ((dict(E=0), 'bad sizes'), (dict(target=0), 'target_samples must be positive'),
                    (dict(ws_bytes=ws - 1), 'workspace too small'), (dict(t_done=None), 'null pointer')):
        a = dict(E=E, target=M * E * 5, t_done=x, ws_bytes=ws)
        a.update(kw)
        rc = lib.promp_paths_finalize_ex(M, a['E'], T, E * T, E * T, 2, 2, a['target'], x, a['t_done'], *([x] * 16), a['ws_bytes'],
                                         None)
        assert rc == ERR and _lib.last_error().startswith('promp_paths_finalize_ex:') and msg in _lib.last_error(), (kw, rc)


# ================================================================================================================ GPU
def _run_fixed(torch, name, reset_mode, M, E, H, shard):
    """Two iterations (update_tasks) of two phases each: [(task params, [phase, phase])] on the host."""
    env, policy, sampler = _sampler(torch, name, M, E, H, reset_mode, shard)
    assert sampler._fused_ok()
    out = []
    for _ in range(2):
        sampler.update_tasks()
        policy.switch_to_pre_update()
        tasks = sampler.vec_env.task_params_per_task.cpu().numpy()
        out.append((tasks, [_fixed_phase(sampler.obtain_samples().phase) for _ in range(2)]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('world', [2, 4])
@pytest.mark.parametrize('reset_mode', ['numpy', 'device'])
@pytest.mark.parametrize('name', FIXED_ENVS)
def test_fixed_horizon_shards_match_global_run(name, reset_mode, world):
    """8 tasks x 5 envs x H = 37 in one sampler vs `world` samplers with task_shard=(r, world): every shard's tasks and
    obs / act / mean / rew / done of both phases of both iterations equal its rows of the global run, bit for bit."""
    torch = _cuda()
    MG, E, H = 8, 5, 37
    M = MG // world
    glob = _run_fixed(torch, name, reset_mode, MG, E, H, None)
    for r in range(world):
        shard = _run_fixed(torch, name, reset_mode, M, E, H, (r, world))
        for it, ((g_tasks, g_phases), (s_tasks, s_phases)) in enumerate(zip(glob, shard)):
            np.testing.assert_array_equal(s_tasks, g_tasks[r * M:(r + 1) * M], err_msg='tasks, iteration %d' % it)
            for p, (g, s) in enumerate(zip(g_phases, s_phases)):
                _assert_fixed_slice(g, s, r, M, 'rank %d/%d iteration %d phase %d' % (r, world, it, p))


def _early_global(torch, name, M, E, H):
    """One phase of the global early-termination run, plus its histogram from promp_paths_histogram."""
    from promp_b200 import _lib
    _, policy, sampler = _sampler(torch, name, M, E, H, 'device', None)
    assert sampler._fused_early_ok()
    sampler.update_tasks()
    policy.update_task_parameters(_task_thetas(torch, name, policy, M))
    ph = sampler.obtain_samples().phase
    T = 2 * H - 1
    hist = torch.zeros(T, dtype=torch.int32, device='cuda')
    _lib.call('promp_paths_histogram', M, E, T, _lib.ptr(ph.timeline['done']), _lib.ptr(hist), _lib.stream())
    return _ragged_phase(ph), hist


def _finalize(torch, tl, target, hist, M, E, T, Do, Da):
    """promp_paths_finalize_ex with histogram `hist` (None: promp_paths_finalize) on host timelines, into zeroed outputs.
    Returns the host outputs, hist afterwards and the workspace afterwards."""
    from promp_b200 import _lib
    from promp_b200.samplers.device_data import DeviceRaggedPhaseData
    d = {k: torch.from_numpy(np.ascontiguousarray(tl['tl_' + k])).cuda() for k in ('obs', 'act', 'mean', 'rew', 'done')}
    n_alloc = (E * T + 3) // 4 * 4
    ph = DeviceRaggedPhaseData(M, E * T, n_alloc, Do, Da, 'cuda')
    for k in ('obs', 'act', 'mean', 'rew', 'done'):
        getattr(ph, k).zero_()
    ws = torch.zeros(_lib.load().promp_paths_workspace_bytes(M, E, T) // 4, dtype=torch.int32, device='cuda')
    p = _lib.ptr
    head = (M, E, T, E * T, n_alloc, Do, Da, int(target))
    tail = (p(d['done']), p(d['obs']), p(d['act']), p(d['mean']), p(d['rew']), p(ph.path_off), p(ph.n_paths), p(ph.n_valid),
            p(ph.src_slot), p(ph.src_start), p(ph.obs), p(ph.act), p(ph.mean), p(ph.rew), p(ph.done), p(ph.cut), p(ws),
            ws.numel() * 4, _lib.stream())
    if hist is None:
        _lib.call('promp_paths_finalize', *head, *tail)
    else:
        _lib.call('promp_paths_finalize_ex', *head, p(hist), *tail)
    out = {k: getattr(ph, k).cpu().numpy() for k in ('cut', 'n_paths', 'n_valid', 'path_off', 'src_slot', 'src_start', 'obs',
                                                      'act', 'mean', 'rew', 'done')}
    out.update({'tl_' + k: np.asarray(tl['tl_' + k]) for k in ('obs', 'act', 'mean', 'rew', 'done')})
    return out, (None if hist is None else hist.cpu().numpy()), ws.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize('world', [2, 3])
@pytest.mark.parametrize('name', EARLY_ENVS)
def test_early_termination_shards_match_global_run(name, world, monkeypatch):
    """6 tasks x 8 envs x H = 40, reset_mode='device', per-task parameters.  Each shard's timelines equal the global slice; the shards'
    histograms sum to the global one; promp_paths_finalize_ex on each shard with the summed histogram and the global target
    reproduces the global run's slice (cut, path table, compacted rows) bit for bit and leaves the histogram and the
    workspace as they were; and so does the sampler itself, with its histogram exchange handing back the global
    histogram."""
    torch = _cuda()
    from promp_b200.utils import dist
    MG, E, H = 6, 8, 40
    T, M = 2 * H - 1, MG // world
    glob, g_hist = _early_global(torch, name, MG, E, H)
    assert glob['cut'][1] == 1
    g_hist_host = g_hist.cpu().numpy()
    local_hists = []

    def exchange(t):        # the sum over ranks, as the all-reduce would give it
        local_hists.append(t.cpu().numpy().copy())
        t.copy_(g_hist)
        return t
    monkeypatch.setattr(dist, 'allreduce_sum_', exchange)
    shards = []
    for r in range(world):
        env, policy, sampler = _sampler(torch, name, M, E, H, 'device', (r, world))
        sampler.update_tasks()
        policy.update_task_parameters(_task_thetas(torch, name, policy, MG)[r * M:(r + 1) * M].contiguous())
        ph = sampler.obtain_samples().phase
        shards.append(_ragged_phase(ph))
        assert len(local_hists) == r + 1
        _assert_ragged_slice(glob, shards[-1], r, M, 'sampler, rank %d/%d' % (r, world))
        assert not sampler._timeline['ws'].any()
    np.testing.assert_array_equal(np.sum(local_hists, axis=0), g_hist_host)
    summed = torch.from_numpy(np.sum(local_hists, axis=0).astype(np.int32)).cuda()
    Do, Da = glob['obs'].shape[-1], glob['act'].shape[-1]
    for r, s in enumerate(shards):
        out, hist_after, ws_after = _finalize(torch, s, MG * E * H, summed, M, E, T, Do, Da)
        _assert_ragged_slice(glob, out, r, M, 'finalize_ex, rank %d/%d' % (r, world))
        np.testing.assert_array_equal(hist_after, g_hist_host)
        assert not ws_after.any()


@pytest.mark.gpu
def test_local_cut_differs_from_global_cut():
    """The cases above exercise the global rule: in the point case, at W = 2 and at W = 3, some shard's own first crossing
    of its local target M*E*H lies at another step than the global t*, so a per-shard cut would keep other paths."""
    torch = _cuda()
    from test_paths_finalize import collect_until
    MG, E, H = 6, 8, 40
    differing = []
    for name in EARLY_ENVS:
        glob, _ = _early_global(torch, name, MG, E, H)
        done = glob['tl_done'].astype(bool)
        t_star = collect_until(done, MG * E * H).t_star
        assert t_star == glob['cut'][0]
        local = {(w, r): collect_until(done[r * (MG // w):(r + 1) * (MG // w)], (MG // w) * E * H).t_star
                 for w in (2, 3) for r in range(w)}
        differing += [(name, w, r, t, t_star) for (w, r), t in local.items() if t != t_star]
    assert {('point', 2), ('point', 3)} <= {d[:2] for d in differing}, differing


@pytest.mark.gpu
def test_ex_entry_points_at_offset_zero_are_the_base_ones():
    """promp_rollout_ex / promp_rollout_early_term_ex with task_offset 0 write what promp_rollout /
    promp_rollout_early_term write, bit for bit; promp_paths_finalize_ex with the histogram promp_paths_histogram builds is
    promp_paths_finalize, and leaves that histogram unchanged; a nonzero offset changes the draws."""
    torch = _cuda()
    from promp_b200 import _lib
    p = _lib.ptr
    M, E, H = 3, 5, 37
    for name in ('point_corner', 'cheetah', 'walker_vel'):
        _, policy, sampler = _sampler(torch, name, M, E, H, 'device', None)
        sampler.update_tasks()
        policy.switch_to_pre_update()
        s = sampler.spec
        params, stride, clip = policy.sampling_params()
        Do, Da = s['obs_dim'], s['act_dim']
        f = lambda *sh: torch.full(sh, float('nan'), device='cuda')
        outs = []
        for entry, off in (('promp_rollout', None), ('promp_rollout_ex', 0), ('promp_rollout_ex', 1)):
            o = dict(obs=f(M, E, H, Do), act=f(M, E, H, Da), mean=f(M, E, H, Da), rew=f(M, E, H), info=f(3, M, E, H), ls=f(M, Da),
                     done=torch.zeros(M, E, H, dtype=torch.uint8, device='cuda'))
            args = (s['env_kind'], s['reward_type'], s['radius'], 1, M, E, H, policy.hidden_arg, p(params), stride,
                    p(sampler.vec_env.task_params_per_task), None, None, PHILOX_SEED, 3, None, clip, float(policy.min_log_std),
                    p(o['obs']), p(o['act']), p(o['mean']), p(o['rew']), p(o['done']), p(o['info']), p(o['ls']), None,
                    _lib.stream())
            _lib.call(entry, *args, *(() if off is None else (off,)))
            outs.append({k: v.cpu().numpy() for k, v in o.items()})
        for k in outs[0]:
            assert np.array_equal(_bits(outs[0][k]), _bits(outs[1][k])), (name, k)
        assert not np.array_equal(_bits(outs[0]['obs']), _bits(outs[2]['obs'])), name

    for name in ('point', 'walker_direc'):
        _, policy, sampler = _sampler(torch, name, M, E, H, 'device', None)
        sampler.update_tasks()
        policy.switch_to_pre_update()
        s = sampler.spec
        params, stride, clip = policy.sampling_params()
        Do, Da, T = s['obs_dim'], s['act_dim'], 2 * H - 1
        f = lambda *sh: torch.full(sh, float('nan'), device='cuda')
        outs = []
        for entry, off in (('promp_rollout_early_term', None), ('promp_rollout_early_term_ex', 0)):
            o = dict(obs=f(M, E, T, Do), act=f(M, E, T, Da), mean=f(M, E, T, Da), rew=f(M, E, T), ls=f(M, Da),
                     done=torch.zeros(M, E, T, dtype=torch.uint8, device='cuda'))
            args = (s['env_kind'], 1, M, E, T, H, policy.hidden_arg, p(params), stride, p(sampler.vec_env.task_params_per_task),
                    None, None, PHILOX_SEED, 3, None, clip, float(policy.min_log_std), p(o['obs']), p(o['act']), p(o['mean']),
                    p(o['rew']), p(o['done']), p(o['ls']), _lib.stream())
            _lib.call(entry, *args, *(() if off is None else (off,)))
            outs.append({k: v.cpu().numpy() for k, v in o.items()})
        for k in outs[0]:
            assert np.array_equal(_bits(outs[0][k]), _bits(outs[1][k])), (name, k)
        # finalize: the workspace histogram vs promp_paths_histogram + finalize_ex, same outputs
        tl = {'tl_' + k: outs[0][k] for k in ('obs', 'act', 'mean', 'rew', 'done')}
        done = torch.from_numpy(outs[0]['done']).cuda()
        hist = torch.zeros(T, dtype=torch.int32, device='cuda')
        _lib.call('promp_paths_histogram', M, E, T, p(done), p(hist), _lib.stream())
        hist_before = hist.cpu().numpy().copy()
        assert int(hist_before.sum()) == int(np.sum(_completed_lengths(outs[0]['done'])))
        got, hist_after, ws = _finalize(torch, tl, M * E * H, hist, M, E, T, Do, Da)
        want, _, ws_base = _finalize(torch, tl, M * E * H, None, M, E, T, Do, Da)
        np.testing.assert_array_equal(hist_after, hist_before)
        assert not ws.any() and not ws_base.any()
        for k in ('cut', 'n_paths', 'n_valid', 'path_off', 'src_slot', 'src_start', 'obs', 'act', 'mean', 'rew', 'done'):
            assert np.array_equal(_bits(got[k]), _bits(want[k])), (name, k)


def _completed_lengths(done):
    """Lengths of the completed paths of [M, E, T] timelines."""
    out = []
    for row in done.reshape(-1, done.shape[-1]):
        ends = np.flatnonzero(row)
        out.extend(np.diff(np.concatenate([[-1], ends])))
    return out


# ================================================================================================================ 2 GPUs
# (env, reset_mode, global tasks, envs per task, horizon): Walker2d early termination runs eagerly, the corner point env
# with host reset draws replays as a CUDA graph (Trainer's default for it)
TWO_GPU = {'walker_device_eager': ('walker_vel', 'device', 4, 8, 40), 'corner_numpy_graph': ('point_corner', 'numpy', 8, 5, 37)}


def _trainer_run(torch, setting, shard):
    """Trainer.train(): ProMP, 2 iterations.  Returns the first phase's samples (host) and the final meta-parameters."""
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    logger.set_quiet(True)
    name, reset_mode, MG, E, H = TWO_GPU[setting]
    M = MG // (shard[1] if shard else 1)
    env, policy, sampler = _sampler(torch, name, M, E, H, reset_mode, shard)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                 clip_eps=0.3, target_inner_step=0.01, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=2, num_inner_grad_steps=1)
    first = {}
    if trainer.graph_capturable():
        capture = trainer.capture_graph

        def capture_recording(*a, **kw):
            step = capture(*a, **kw)

            def recording_step(*sa, **skw):
                phases = step(*sa, **skw)
                if not first:
                    first.update(_fixed_phase(phases[0]))
                return phases
            return recording_step
        trainer.capture_graph = capture_recording
    else:
        obtain = sampler.obtain_samples

        def recording_obtain(*a, **kw):
            paths = obtain(*a, **kw)
            if not first:
                first.update(_ragged_phase(paths.phase) if hasattr(paths.phase, 'cut') else _fixed_phase(paths.phase))
            return paths
        sampler.obtain_samples = recording_obtain
    trainer.train()
    torch.cuda.synchronize()
    return first, policy.theta.cpu().numpy().copy()


def _worker_main(setting, out_dir):
    import datetime
    import torch
    import torch.distributed as dist
    from promp_b200.utils.dist import enable_p2p_allreduce
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    torch.cuda.set_device(int(os.environ['LOCAL_RANK']))
    dist.init_process_group('nccl', device_id=torch.device('cuda', torch.cuda.current_device()),
                            timeout=datetime.timedelta(seconds=60))
    enable_p2p_allreduce()
    first, theta = _trainer_run(torch, setting, (rank, world))
    np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), theta=theta, **first)
    dist.barrier()
    dist.destroy_process_group()
    print("rank %d sharded ok" % rank)


@pytest.mark.gpu
@pytest.mark.parametrize('setting', list(TWO_GPU))
def test_two_gpus_match_one_process(setting, tmp_path):
    """Trainer.train() (ProMP, 2 iterations) at world 2 vs one process with the global batch: each rank's first phase is
    its slice of the global one, bit for bit; the meta-parameters after 2 iterations agree within 1e-5 relative (the
    meta-gradient all-reduce sums in another order)."""
    torch = _cuda()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = 29561 + list(TWO_GPU).index(setting)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(port), os.path.abspath(__file__), setting, str(tmp_path)]
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=200)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)        # the launcher and both workers
        out, _ = proc.communicate()
        pytest.fail("2-rank run timed out:\n" + out[-3000:])
    assert proc.returncode == 0 and 'rank 0 sharded ok' in out and 'rank 1 sharded ok' in out, out[-3000:]
    torch.cuda.set_device(0)
    glob, theta = _trainer_run(torch, setting, None)
    M = TWO_GPU[setting][2] // 2
    for r in range(2):
        got = dict(np.load(os.path.join(str(tmp_path), 'rank%d.npz' % r)))
        t_r = got.pop('theta')
        if 'cut' in glob:
            _assert_ragged_slice(glob, got, r, M, 'rank %d' % r)
        else:
            _assert_fixed_slice(glob, got, r, M, 'rank %d' % r)
        rel = np.linalg.norm(t_r - theta) / np.linalg.norm(theta)
        assert rel < 1e-5, (r, rel)


if __name__ == '__main__':
    _worker_main(sys.argv[1], sys.argv[2])
