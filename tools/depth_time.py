"""Policies with one, two and three hidden layers of 64 units on the H100: kernel time of the gradient, Hessian-vector,
forward and fused rollout kernels, and ms per ProMP meta-iteration replayed as one CUDA graph.  Prints the card name, power
limit and maximum SM clock with the numbers.

Kernels: tools/activation_time.py's calls (CUDA events, 5 warm-up + 30 timed launches) plus promp_policy_forward on the same
N = E*H observations per task, tanh hidden layers of 64 units, at PointEnvCorner (obs 2, act 2) 40 x 20 x 100 and the cheetah
surrogate (obs 17, act 6) 40 x 20 x 200; the three depths alternated `--repeats` times.  Depth 2 runs the tensor-core
gradient / HVP kernels (the default), depths 1 and 3 the CUDA-core kernels of policy_deep.cuh.  Trainer: the BASELINE.json
configs[1] (PointEnv 40 x 20 x 100) and configs[2] (cheetah surrogate 40 x 20 x 200) sizes, ProMP with one inner step and 5
Adam epochs, captured once and replayed `--warmup` + `--itrs` times.  [min, max] = the spread over the repeats.

usage: python tools/depth_time.py [--repeats 3] [--itrs 10] [--warmup 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from promp_b200 import _lib  # noqa: E402
from activation_time import WORKLOADS, _timeit, kernel_calls  # noqa: E402

DEPTHS = (1, 2, 3)


def forward_call(wl, hidden_arg, M=40, E=20):
    _, Do, Da, _, H = WORKLOADS[wl]
    N = E * H
    P = _lib.load().promp_num_params(Do, Da, hidden_arg)
    g = torch.Generator(device='cuda').manual_seed(1)
    theta = (0.1 * torch.randn(M, P, generator=g, device='cuda')).contiguous()
    obs = torch.randn(M, N, Do, generator=g, device='cuda')
    mean = torch.empty(M, N, Da, device='cuda')
    p = _lib.ptr
    return lambda: _lib.call('promp_policy_forward', Do, Da, hidden_arg, M, N, p(theta), P, p(obs), p(mean), _lib.stream())


def graph_ms(wl, depth, itrs, warmup, M=40, E=20):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnvCorner, HalfCheetahRandDirecEnv
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.utils import logger
    logger.set_quiet(True)
    np.random.seed(3)
    _, Do, Da, _, H = WORKLOADS[wl]
    env = normalize(MetaPointEnvCorner() if wl == 'point' else HalfCheetahRandDirecEnv())
    policy = MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64,) * depth)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=True)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=warmup + itrs,
                      num_inner_grad_steps=1, use_cuda_graph=True)
    step = trainer.capture_graph(log=False)
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(itrs):
        step(warmup + i)
    b.record()
    torch.cuda.synchronize()
    assert torch.isfinite(policy.theta).all()
    return a.elapsed_time(b) / itrs


def _stats(v):
    return dict(mean=float(np.mean(v)), min=float(np.min(v)), max=float(np.max(v)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--itrs', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _lib.require_cuda()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    res = dict(card=card, kernels_us={}, graph_ms={})
    for wl in WORKLOADS:
        calls = {}
        for d in DEPTHS:
            h = 64 | _lib.hidden_depth(d)
            calls[d] = dict(kernel_calls(wl, h), forward=forward_call(wl, h))
        for k in ('grad', 'hvp', 'forward', 'rollout'):
            runs = {d: [] for d in DEPTHS}
            for _ in range(a.repeats):
                for d in DEPTHS:
                    runs[d].append(_timeit(calls[d][k]))
            res['kernels_us']['%s/%s' % (wl, k)] = {str(d): _stats(v) for d, v in runs.items()}
        runs = {d: [] for d in DEPTHS}
        for _ in range(a.repeats):
            for d in DEPTHS:
                runs[d].append(graph_ms(wl, d, a.itrs, a.warmup))
        res['graph_ms'][wl] = {str(d): _stats(v) for d, v in runs.items()}
    print('card: %s' % card)
    rows = list(res['kernels_us'].items()) + [('%s/ProMP ms' % wl, v) for wl, v in res['graph_ms'].items()]
    for key, v in rows:
        print('  %-18s' % key + ''.join('   depth %s %9.2f [%.2f, %.2f]' % (d, v[d]['mean'], v[d]['min'], v[d]['max'])
                                       for d in map(str, DEPTHS)))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'depth_time.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
