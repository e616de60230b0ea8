"""Time the Walker2d and Swimmer surrogates at 40 tasks x 20 envs x H = 200 (hidden 64, normalize(env)):
  * the fused rollout (promp_rollout; the walker's fixed-horizon record) per sampling phase;
  * one ProMP meta-iteration through Trainer.train() (CUDA-graph mode where the trainer selects it);
  * walker: MetaSampler(reset_mode='device') (fused early termination + device path table) against 'numpy' (the
    reference's step loop with host reset draws), per sampling phase and per meta-iteration.
Prints the card name and its power limit, read in the same run.

    python tools/locomotion_time.py [--iters K] [--warmup W]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200.baselines import LinearFeatureBaseline  # noqa: E402
from promp_b200.envs import normalize, Walker2DRandVelEnv, SwimmerRandVelEnv  # noqa: E402
from promp_b200.meta_algos import ProMP  # noqa: E402
from promp_b200.meta_trainer import Trainer  # noqa: E402
from promp_b200.policies import MetaGaussianMLPPolicy  # noqa: E402
from promp_b200.samplers import MetaSampler, MetaSampleProcessor  # noqa: E402
from promp_b200.samplers.device_data import PhaseData  # noqa: E402
from promp_b200.utils import logger  # noqa: E402

M, E, H = 40, 20, 200


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=power.limit',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out


def stack(env_cls, reset_mode, seed=1):
    np.random.seed(seed)
    env = normalize(env_cls())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=env.obs_dim, action_dim=env.act_dim, meta_batch_size=M,
                                   hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H,
                          reset_mode=reset_mode, seed=seed)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    return env, policy, sampler, proc, algo


def time_cuda(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def time_wall(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters * 1e3


def rollout_ms(env_cls, iters, warmup):
    env, policy, sampler, _, _ = stack(env_cls, 'device')
    sampler.update_tasks()
    policy.switch_to_pre_update()
    ph = PhaseData(M, E, H, env.obs_dim, env.act_dim, sampler.device)
    return time_cuda(lambda: sampler.rollout_into(ph), iters, warmup)


def sampling_ms(env_cls, reset_mode, iters, warmup):
    env, policy, sampler, _, _ = stack(env_cls, reset_mode)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    return time_wall(sampler.obtain_samples, iters, warmup)


def meta_iteration_ms(env_cls, reset_mode, iters, warmup):
    env, policy, sampler, proc, algo = stack(env_cls, reset_mode)
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=warmup,
                      num_inner_grad_steps=1)
    trainer.train()                                   # warm-up iterations (graph capture, if selected, happens here)
    trainer.start_itr, trainer.n_itr = warmup, warmup + iters
    torch.cuda.synchronize()
    t = time.perf_counter()
    trainer.train()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters * 1e3, trainer.graph_capturable()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    logger.set_quiet(True)
    name, plimit = card()
    print('card: %s, power limit %s' % (name, plimit))
    print('M x E x H = %d x %d x %d, hidden 64' % (M, E, H))
    for env_cls in (Walker2DRandVelEnv, SwimmerRandVelEnv):
        n = env_cls.__name__
        print('%-20s rollout (promp_rollout)               %8.3f ms per phase' % (n, rollout_ms(env_cls, args.iters, args.warmup)))
        if env_cls is Walker2DRandVelEnv:
            for mode in ('device', 'numpy'):
                k = args.iters if mode == 'device' else max(1, args.iters // 5)
                print('%-20s sampling, reset_mode=%-6s            %8.3f ms per phase'
                      % (n, mode, sampling_ms(env_cls, mode, k, 1)))
            for mode in ('device', 'numpy'):
                k = args.iters if mode == 'device' else max(1, args.iters // 5)
                ms, graph = meta_iteration_ms(env_cls, mode, k, 1 if mode == 'numpy' else args.warmup)
                print('%-20s ProMP meta-iteration, reset_mode=%-6s %8.3f ms (graph mode: %s)' % (n, mode, ms, graph))
        else:
            ms, graph = meta_iteration_ms(env_cls, 'numpy', args.iters, args.warmup)
            print('%-20s ProMP meta-iteration                   %8.3f ms (graph mode: %s)' % (n, ms, graph))


if __name__ == '__main__':
    main()
