"""Timings of users' own environments (promp_b200.envs.CudaMetaEnv), on the GPU:
  - JIT: cold (empty cache) and warm (disk cache) compile time of one policy variant;
  - twin vs built-in rollout kernel time (PointCorner fixed horizon, Walker early termination), CUDA events;
  - cart-pole sampling phase: fused early-termination kernel + path table vs the stepwise env-step loop;
  - one ProMP meta-iteration on the pendulum replayed as a CUDA graph.
Usage: python tools/cuda_env_time.py [--reps 50] [--out results/cuda_env_time.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def ev_time(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3)
    return float(np.median(out)), float(np.min(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    os.environ['PROMP_B200_JIT_CACHE'] = tempfile.mkdtemp(prefix='promp_jit_time_')
    import torch
    from promp_b200 import _jit
    from promp_b200.envs import normalize
    from promp_b200.utils import logger
    import test_cuda_envs as T
    logger.set_quiet(True)
    torch.cuda.set_device(0)
    res = dict(gpu=torch.cuda.get_device_name(0), nvrtc='%d.%d' % _jit.nvrtc().version,
               nvrtc_matches_library=_jit.matches_library())

    # ---- JIT: cold then warm, one variant (env kernels + keyed / unkeyed rollout), the walker twin and the pendulum
    for name, make in (('walker_twin', lambda: T._twin('walker')[1]), ('pendulum', T.make_pendulum)):
        t = time.perf_counter()
        env = make()
        env.program.kernels(64)
        cold = time.perf_counter() - t
        t = time.perf_counter()
        env = make()
        env.program.kernels(64)
        res['jit_%s_cold_s' % name], res['jit_%s_warm_s' % name] = cold, time.perf_counter() - t

    # ---- twin vs built-in rollout
    M, E, H = 40, 20, 100
    for kind in ('point', 'walker'):
        inner, twin = T._twin(kind)
        Hk = H if kind == 'point' else 200
        for label, env in (('builtin', normalize(inner)), ('twin', normalize(twin))):
            policy, sampler = T._sampler(torch, env, M, E, Hk)
            if kind == 'point':
                from promp_b200.samplers.device_data import PhaseData
                ph = PhaseData(M, E, Hk, env.obs_dim, env.act_dim, sampler.device)
                fn = lambda: sampler.rollout_into(ph)       # noqa: E731
            else:
                fn = sampler.obtain_samples      # early-term kernel + path table
            res['rollout_%s_%s_us' % (kind, label)] = ev_time(torch, fn, args.reps)

    # ---- cart-pole phase: fused vs stepwise
    env = normalize(T.make_cartpole())
    policy, sampler = T._sampler(torch, env, M, E, H, reset_mode='device')
    res['cartpole_phase_fused_us'] = ev_time(torch, sampler.obtain_samples, args.reps)
    policy, sampler = T._sampler(torch, env, M, E, H, reset_mode='numpy')
    t = time.perf_counter()
    sampler.obtain_samples()
    torch.cuda.synchronize()
    res['cartpole_phase_stepwise_ms'] = (time.perf_counter() - t) * 1e3

    # ---- one ProMP meta-iteration on the pendulum, graph replay
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.samplers import MetaSampleProcessor
    env = normalize(T.make_pendulum())
    policy, sampler = T._sampler(torch, env, M, E, H, reset_mode='device')
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, learning_rate=1e-3, num_ppo_steps=5,
                 clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    tr = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=1, num_inner_grad_steps=1,
                 use_cuda_graph=True)
    step = tr.capture_graph()
    res['promp_pendulum_graph_iter_us'] = ev_time(torch, step, args.reps)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
