"""Identity vs tanh output layer on the H100: kernel time of the gradient, Hessian-vector and fused rollout kernels, and ms per
eager ProMP meta-iteration through Trainer.train_iteration().  Prints the card name, power limit and maximum SM clock with
the numbers.

Kernels: tools/activation_time.py's calls (CUDA events, 5 warm-up + 30 timed launches) with tanh hidden layers of 64 units,
`hidden` = 64 (identity output) and 64 | PROMP_OUT_TANH, alternated `--repeats` times, at PointEnvCorner (obs 2, act 2)
40 x 20 x 100 and the cheetah (obs 17, act 6) 40 x 20 x 200.  Trainer: ProMP, one inner step, 5 Adam epochs, M = 40,
E = 20, H = 100 on the point env; the mean ms of iterations 2..n.  The [min, max] beside each mean is the spread over the
repeats.

usage: python tools/output_tanh_time.py [--repeats 5] [--itrs 6] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from promp_b200 import _lib  # noqa: E402
from activation_time import WORKLOADS, _timeit, kernel_calls  # noqa: E402

OUTPUTS = (None, 'tanh')


def _label(out):
    return 'identity' if out is None else 'tanh'


def trainer_ms(out, itrs, M=40, E=20, H=100):
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, MetaPointEnvCorner
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.utils import logger
    logger.set_quiet(True)
    np.random.seed(3)
    env = normalize(MetaPointEnvCorner())
    policy = MetaGaussianMLPPolicy(name='p', obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64),
                                   output_nonlinearity=out)
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=itrs,
                      num_inner_grad_steps=1)
    times = []
    for itr in range(itrs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        trainer.train_iteration(itr, log=True)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        logger.dumpkvs()
    return float(np.mean(times[2:]))


def _stats(v):
    return dict(mean=float(np.mean(v)), min=float(np.min(v)), max=float(np.max(v)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--itrs', type=int, default=6)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _lib.require_cuda()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    res = dict(card=card, kernels_us={}, trainer_ms={})
    calls = {(wl, out): kernel_calls(wl, 64 | (_lib.OUT_TANH if out else 0)) for wl in WORKLOADS for out in OUTPUTS}
    for wl in WORKLOADS:
        for k in ('grad', 'hvp', 'rollout'):
            runs = {out: [] for out in OUTPUTS}
            for _ in range(a.repeats):
                for out in OUTPUTS:
                    runs[out].append(_timeit(calls[(wl, out)][k]))
            res['kernels_us']['%s/%s' % (wl, k)] = {_label(out): _stats(v) for out, v in runs.items()}
    runs = {out: [] for out in OUTPUTS}
    for _ in range(max(1, a.repeats - 2)):
        for out in OUTPUTS:
            runs[out].append(trainer_ms(out, a.itrs))
    res['trainer_ms'] = {_label(out): _stats(v) for out, v in runs.items()}
    print('card: %s' % card)
    for key, v in list(res['kernels_us'].items()) + [('ProMP iteration ms', res['trainer_ms'])]:
        print('  %-20s identity %8.2f [%.2f, %.2f]   tanh %8.2f [%.2f, %.2f]' % (
            key, v['identity']['mean'], v['identity']['min'], v['identity']['max'], v['tanh']['mean'], v['tanh']['min'],
            v['tanh']['max']))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'output_tanh_time.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
