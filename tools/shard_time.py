"""Per-phase time of early-termination sampling (Walker2d surrogate, reset_mode='device', M x E x H = 40 x 20 x 200 per
GPU), with the cut taken two ways:
  local   promp_rollout_early_term + promp_paths_finalize (the cut from the launch's own histogram: one process)
  global  promp_rollout_early_term_ex + promp_paths_histogram + promp_paths_finalize_ex (the cut from a caller's
          histogram: what a sharded MetaSampler runs), at world 1 without an exchange
and, on a machine with two GPUs, `global` at world 2 with the NCCL all-reduce of the int32 histogram between the two
stages (the script relaunches itself under torch.distributed.run).  CUDA events over --iters phases after --warmup, the
two single-GPU variants alternated --reps times.  Prints the card name and power limit with the numbers.
usage: python tools/shard_time.py [--iters 50] [--warmup 10] [--reps 3]"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
M, E, H = 40, 20, 200


def _setup(shard):
    import torch
    from promp_b200 import _lib
    from promp_b200.envs import normalize, Walker2DRandVelEnv
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler
    np.random.seed(1)
    env = normalize(Walker2DRandVelEnv())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=env.obs_dim, action_dim=env.act_dim, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          reset_mode='device', seed=1, task_shard=shard)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    ph = sampler.obtain_samples().phase            # allocates the timelines and the workspace
    world = shard[1] if shard else 1
    offset = shard[0] * M if shard else 0
    s, tl, p = sampler.spec, sampler._timeline, _lib.ptr
    T, Do, Da = 2 * H - 1, s['obs_dim'], s['act_dim']
    n_alloc = (E * T + 3) // 4 * 4
    params, stride, clip = policy.sampling_params()
    hist = torch.zeros(T, dtype=torch.int32, device='cuda')
    counter = [100]

    def rollout(entry, *extra):
        counter[0] += 1
        _lib.call(entry, s['env_kind'], 1, M, E, T, H, policy.hidden_arg, p(params), stride, p(sampler.vec_env.task_params_per_task),
                  None, None, 1, counter[0], None, clip, float(policy.min_log_std), p(tl['obs']), p(tl['act']), p(tl['mean']),
                  p(tl['rew']), p(tl['done']), p(ph.log_std), _lib.stream(), *extra)

    head = (M, E, T, E * T, n_alloc, Do, Da)
    tail = (p(tl['done']), p(tl['obs']), p(tl['act']), p(tl['mean']), p(tl['rew']), p(ph.path_off), p(ph.n_paths), p(ph.n_valid),
            p(ph.src_slot), p(ph.src_start), p(ph.obs), p(ph.act), p(ph.mean), p(ph.rew), p(ph.done), p(ph.cut), p(tl['ws']),
            tl['ws'].numel() * 4, _lib.stream())

    def local_cut():
        rollout('promp_rollout_early_term')
        _lib.call('promp_paths_finalize', *head, M * E * H, *tail)

    def global_cut(exchange=None):
        rollout('promp_rollout_early_term_ex', offset)
        hist.zero_()
        _lib.call('promp_paths_histogram', M, E, T, p(tl['done']), p(hist), _lib.stream())
        if exchange is not None:
            exchange(hist)
        _lib.call('promp_paths_finalize_ex', *head, world * M * E * H, p(hist), *tail)
    return local_cut, global_cut


def _time(fn, iters, warmup, sync=None):
    import torch
    for _ in range(warmup):
        fn()
    (sync or torch.cuda.synchronize)()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return r.stdout.strip() or 'unknown card'


def _worker(args):
    import datetime
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    torch.cuda.set_device(int(os.environ['LOCAL_RANK']))
    dist.init_process_group('nccl', device_id=torch.device('cuda', torch.cuda.current_device()),
                            timeout=datetime.timedelta(seconds=60))
    _, global_cut = _setup((rank, world))
    exchange = lambda h: dist.all_reduce(h, op=dist.ReduceOp.SUM)
    ms = _time(lambda: global_cut(exchange), args.iters, args.warmup, sync=lambda: (torch.cuda.synchronize(), dist.barrier()))
    t = torch.tensor([ms], device='cuda')
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print('world 2, global cut + NCCL histogram all-reduce: %.3f ms per phase (slowest rank)' % float(t.item()))
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return _worker(args)
    import torch
    from promp_b200 import _lib
    _lib.require_cuda()
    print('card: %s' % _card())
    print('Walker2DRandVelEnv, reset_mode=device, M x E x H = %d x %d x %d, timeline 2H-1 = %d steps' % (M, E, H, 2 * H - 1))
    local_cut, global_cut = _setup(None)
    res = {'local': [], 'global': []}
    for _ in range(args.reps):
        res['local'].append(_time(local_cut, args.iters, args.warmup))
        res['global'].append(_time(global_cut, args.iters, args.warmup))
    for k, label in (('local', 'rollout + promp_paths_finalize'),
                     ('global', 'rollout_ex + promp_paths_histogram + promp_paths_finalize_ex')):
        v = res[k]
        print('world 1, %-62s %.3f ms per phase (reps %s)' % (label, float(np.mean(v)), ', '.join('%.3f' % x for x in v)))
    if torch.cuda.device_count() >= 2:
        cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
               '--master-port', '29571', os.path.abspath(__file__), '--worker', '--iters', str(args.iters), '--warmup',
               str(args.warmup)]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
        print(r.stdout.strip() if r.returncode == 0 else 'world 2: failed\n' + r.stdout[-2000:] + r.stderr[-2000:])
    else:
        print('world 2, global cut + NCCL histogram all-reduce: not measured (one GPU visible)')


if __name__ == '__main__':
    main()
