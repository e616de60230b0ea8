"""Fixed vs trainable inner step sizes (Meta-SGD) on the H100: ms per ProMP meta-iteration replayed as one CUDA graph
(Trainer.capture_graph), alternated `--repeats` times.  Prints the card name, power limit and maximum SM clock with the
numbers.

Workloads: ProMP, one inner step, 5 Adam epochs, M = 40 tasks, E = 20 rollouts, at PointEnvCorner (H = 100) and the
HalfCheetahRandDirec surrogate (H = 200).  Each run captures one iteration, replays `--warmup` iterations untimed and then
`--itrs` timed ones between CUDA events; the [min, max] beside each mean is the spread over the repeats.

usage: python tools/meta_sgd_time.py [--repeats 5] [--itrs 10] [--warmup 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200 import _lib  # noqa: E402

WORKLOADS = {'point': (2, 2, 100), 'cheetah': (17, 6, 200)}


def graph_ms(wl, trainable, itrs, warmup, M=40, E=20):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnvCorner, HalfCheetahRandDirecEnv
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.utils import logger
    logger.set_quiet(True)
    np.random.seed(3)
    Do, Da, H = WORKLOADS[wl]
    env = normalize(MetaPointEnvCorner() if wl == 'point' else HalfCheetahRandDirecEnv())
    policy = MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=True, trainable_inner_step_size=trainable)
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
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--itrs', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _lib.require_cuda()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    res = dict(card=card, graph_ms={})
    for wl in WORKLOADS:
        runs = {False: [], True: []}
        for _ in range(a.repeats):
            for trainable in (False, True):
                runs[trainable].append(graph_ms(wl, trainable, a.itrs, a.warmup))
        res['graph_ms'][wl] = dict(fixed=_stats(runs[False]), trainable=_stats(runs[True]))
    print('card: %s' % card)
    for wl, v in res['graph_ms'].items():
        f, t = v['fixed'], v['trainable']
        print('  %-8s fixed %8.3f [%.3f, %.3f] ms   trainable %8.3f [%.3f, %.3f] ms   (%+.1f %%)' % (
            wl, f['mean'], f['min'], f['max'], t['mean'], t['min'], t['max'], 100.0 * (t['mean'] / f['mean'] - 1.0)))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'meta_sgd_time.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
