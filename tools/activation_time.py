"""Tanh vs ReLU policies on the H100: kernel time of the gradient, Hessian-vector and fused rollout kernels, and ms per ProMP
meta-iteration through Trainer.train().  Prints the card name and power limit with the numbers.

Kernels (CUDA events, 5 warm-up + 30 timed launches, L2-warm like the training loop), the two activations alternated
`--repeats` times, at PointEnvCorner (obs 2, act 2) and the cheetah (obs 17, act 6) with M x E x H = 40 x 20 x H
(H = 100 point, 200 cheetah: N = E*H samples per task):
    grad   promp_policy_grad, per-task parameters, RATIO objective
    hvp    promp_policy_hvp, per-task parameters
    rollout promp_rollout, pre-update parameters, in-kernel reset states and noise
Trainer: ProMP with one inner step (5 Adam epochs), M = 40, E = 20, H = 100 on the point env, eager mode; the mean ms of
iterations 2..n (the first two allocate the device buffers and workspaces).

usage: python tools/activation_time.py [--repeats 3] [--itrs 6] [--out DIR]
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
from promp_b200 import _lib  # noqa: E402

WORKLOADS = dict(point=(_lib.ENV_POINT_CORNER, 2, 2, 2, 100), cheetah=(_lib.ENV_CHEETAH_DIR, 17, 6, 1, 200))


def _timeit(fn, n=30):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3


def kernel_calls(wl, hidden_arg, M=40, E=20):
    kind, Do, Da, TD, H = WORKLOADS[wl]
    N = E * H
    P = _lib.load().promp_num_params(Do, Da, hidden_arg)
    dev = torch.device('cuda')
    g = torch.Generator(device='cuda').manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    theta_t = (0.1 * r(P)).view(1, -1).repeat(M, 1).contiguous()
    obs, act, adv, mean, ls = r(M, N, Do), r(M, N, Da), r(M, N), r(M, N, Da), 0.1 * r(M, Da)
    grad, newp, vec, out = torch.empty(M, P, device=dev), torch.empty(M, P, device=dev), 0.01 * r(M, P), torch.empty(M, P, device=dev)
    st = torch.zeros(M, 4, device=dev)
    need = _lib.load().promp_policy_workspace_bytes(M, N, Do, Da, hidden_arg)
    ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device=dev)
    task = torch.ones(M, TD, device=dev)
    r_obs, r_act, r_mean = torch.empty(M, E, H, Do, device=dev), torch.empty(M, E, H, Da, device=dev), torch.empty(M, E, H, Da, device=dev)
    r_rew, r_done = torch.empty(M, E, H, device=dev), torch.empty(M, E, H, dtype=torch.uint8, device=dev)
    r_info, r_ls = torch.empty(3, M, E, H, device=dev), torch.empty(M, Da, device=dev)
    p, s = _lib.ptr, _lib.stream()

    def grad_call():
        _lib.call('promp_policy_grad', Do, Da, hidden_arg, M, N, p(theta_t), P, p(obs), p(act), p(adv), p(mean), p(ls), 0, 0, 1.0,
                  0.3, 0.0, 0, -13.8, p(grad), p(newp), 0.1, p(st), p(ws), ws.numel() * 4, s)

    def hvp_call():
        _lib.call('promp_policy_hvp', Do, Da, hidden_arg, M, N, p(theta_t), P, p(obs), p(act), p(adv), p(mean), p(ls), 0, 0, 0.1,
                  5e-4, 0, -13.8, p(vec), p(out), p(st), p(ws), ws.numel() * 4, s)

    def rollout_call():
        _lib.call('promp_rollout', kind, 0 if kind == _lib.ENV_CHEETAH_DIR else _lib.REWARD_DENSE, 0.5, 1, M, E, H, hidden_arg,
                  p(theta_t), 0, p(task), None, None, 7, 1, None, 1, -13.8, p(r_obs), p(r_act), p(r_mean), p(r_rew), p(r_done),
                  p(r_info), p(r_ls), None, s)
    return dict(grad=grad_call, hvp=hvp_call, rollout=rollout_call)


def trainer_ms(act, itrs, M=40, E=20, H=100):
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
                                   hidden_nonlinearity=act)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--itrs', type=int, default=6)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    _lib.require_cuda()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    res = dict(card=card, kernels_us={}, trainer_ms={})
    calls = {(wl, act): kernel_calls(wl, 64 | (_lib.ACT_RELU if act == 'relu' else 0)) for wl in WORKLOADS for act in ('tanh', 'relu')}
    for wl in WORKLOADS:
        for k in ('grad', 'hvp', 'rollout'):
            runs = {act: [] for act in ('tanh', 'relu')}
            for _ in range(a.repeats):
                for act in ('tanh', 'relu'):
                    runs[act].append(_timeit(calls[(wl, act)][k]))
            res['kernels_us']['%s/%s' % (wl, k)] = {act: dict(mean=float(np.mean(v)), min=float(np.min(v)), max=float(np.max(v)))
                                                    for act, v in runs.items()}
    runs = {act: [] for act in ('tanh', 'relu')}
    for _ in range(max(1, a.repeats - 1)):
        for act in ('tanh', 'relu'):
            runs[act].append(trainer_ms(act, a.itrs))
    res['trainer_ms'] = {act: dict(mean=float(np.mean(v)), min=float(np.min(v)), max=float(np.max(v))) for act, v in runs.items()}
    print('card: %s' % card)
    for key, v in res['kernels_us'].items():
        print('  %-16s tanh %8.1f us [%.1f, %.1f]   relu %8.1f us [%.1f, %.1f]' % (
            key, v['tanh']['mean'], v['tanh']['min'], v['tanh']['max'], v['relu']['mean'], v['relu']['min'], v['relu']['max']))
    v = res['trainer_ms']
    print('  %-16s tanh %8.2f ms [%.2f, %.2f]   relu %8.2f ms [%.2f, %.2f]' % (
        'ProMP iteration', v['tanh']['mean'], v['tanh']['min'], v['tanh']['max'], v['relu']['mean'], v['relu']['min'], v['relu']['max']))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'activation_time.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
