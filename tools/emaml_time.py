"""E-MAML timing on the reference's e-maml configuration (TRPOMAML(exploration=True), normalize(HalfCheetahRandDirecEnv) surrogate,
M x E x H = 40 x 20 x 100, hidden 64, one inner step):
  iteration  one meta-iteration through the Trainer, eager (train_iteration) against the CUDA-graph replay (capture_graph step)
  loss       one TRPO line-search evaluation (loss_terms_dev): the previous composition - meta pass, then a stand-alone LOGLIK
             launch on the expanded [M, N] coefficient, a sum and an add - against the exploration stage inside the chain
  grad       the meta-gradient the same two ways (previous: + promp_reduce_tasks + add)
Both variants of each pair are alternated --reps times.  CUDA events around --iters evaluations after --warmup (loss, grad);
a host clock around --itr-iters synchronised iterations (iteration).  Also reports whether the two compositions give the
same bits.  Prints the card name and power limit with the numbers.
usage: python tools/emaml_time.py [--iters 200] [--warmup 20] [--itr-iters 5] [--reps 3]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
M, E, H = 40, 20, 100


def _trainer(graph):
    import torch
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.envs import normalize, HalfCheetahRandDirecEnv
    from promp_b200.meta_algos import TRPOMAML
    from promp_b200.meta_trainer import Trainer
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    np.random.seed(1)
    torch.manual_seed(1)
    env = normalize(HalfCheetahRandDirecEnv())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=int(np.prod(env.observation_space.shape)),
                                   action_dim=int(np.prod(env.action_space.shape)), meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = TRPOMAML(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=1, step_size=0.01, exploration=True)
    return Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=10 ** 6, num_inner_grad_steps=1,
                   use_cuda_graph=graph)


def _previous(algo):
    """The loss / gradient evaluations as composed before the exploration stage existed (reproduced for the comparison)."""
    import torch
    from promp_b200 import _lib

    def loss(theta, phases):
        res = algo._meta_pass(theta, phases, _lib.OBJ_RATIO, 0.0, [0.0], want_grad=False)
        out = torch.empty(3, dtype=torch.float32, device='cuda')
        _lib.call('promp_meta_loss_terms', 2, M, _lib.ptr(res['stats_all']), 1.0 / M, None, 3, _lib.ptr(out), _lib.stream())
        st = torch.zeros(M, 4, dtype=torch.float32, device='cuda')
        algo._grad(phases[0], theta, 0, _lib.OBJ_LOGLIK, clip_log_std=1, stats=st, adv=algo._exploration_coeff(phases))
        out[0] += st[:, 0].sum() / M
        return out

    def grad(theta, phases):
        res = algo._meta_pass(theta, phases, _lib.OBJ_RATIO, 0.0, [0.0], want_grad=True)
        st = torch.zeros(M, 4, dtype=torch.float32, device='cuda')
        g = torch.empty(M, algo.policy.num_params, dtype=torch.float32, device='cuda')
        algo._grad(phases[0], theta, 0, _lib.OBJ_LOGLIK, clip_log_std=1, grad=g, stats=st, adv=algo._exploration_coeff(phases))
        extra = torch.empty_like(res['grad'])
        _lib.call('promp_reduce_tasks', M, algo.policy.num_params, _lib.ptr(g), 1.0 / M, _lib.ptr(extra), _lib.stream())
        res['grad'] += extra
        return res['grad']
    return loss, grad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--itr-iters', type=int, default=5)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    import torch
    from promp_b200.utils import logger
    torch.cuda.set_device(0)
    logger.set_quiet(True)
    try:
        card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception:        # noqa: BLE001 - the query is informational
        card = torch.cuda.get_device_name(0)
    print("card: %s" % card)

    # ---- per evaluation: previous composition vs the exploration stage in the chain, on one iteration's phases
    tr = _trainer(False)
    algo, policy = tr.algo, tr.policy
    tr.sampler.update_tasks()
    policy.switch_to_pre_update()
    samples = []
    for step in range(2):
        s = tr.sample_processor.process_samples(tr.sampler.obtain_samples())
        samples.append(s)
        if step == 0:
            algo._adapt(s)
    phases = [s[0].phase for s in samples]
    algo._adapt_cache = None
    theta = policy.theta.clone()
    old_loss, old_grad = _previous(algo)
    variants = dict(loss=(lambda: old_loss(theta, phases), lambda: algo.loss_terms_dev(theta, phases)),
                    grad=(lambda: old_grad(theta, phases), lambda: algo.eval_gradient_dev(theta, phases, 'loss')))
    for name, (f_old, f_new) in variants.items():
        o, n = f_old().clone(), f_new().clone()
        torch.cuda.synchronize()
        print("%s: previous vs new bit-identical: %s, max rel diff %.3g" % (
            name, bool(torch.equal(o, n)), float((o - n).abs().max() / (o.abs().max() + 1e-30))))
    for name, (f_old, f_new) in variants.items():
        res = {'previous': [], 'new': []}
        for _ in range(a.reps):
            for label, f in (('previous', f_old), ('new', f_new)):
                for _ in range(a.warmup):
                    f()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    f()
                e1.record()
                torch.cuda.synchronize()
                res[label].append(1000.0 * e0.elapsed_time(e1) / a.iters)
        for label, v in res.items():
            print("%s %-8s us/evaluation: %s" % (name, label, " ".join("%.1f" % x for x in v)))

    # ---- per meta-iteration: eager vs graph replay
    tr_e, tr_g = _trainer(False), _trainer(True)
    assert tr_g.graph_capturable()
    step = tr_g.capture_graph(warmup=2, log=False)
    for itr in range(2):                     # warm-up of both
        tr_e.train_iteration(itr, log=False)
        step(itr)
    torch.cuda.synchronize()
    res = {'eager': [], 'graph': []}
    itr = 2
    for _ in range(a.reps):
        for label in ('eager', 'graph'):
            t0 = time.perf_counter()
            for _ in range(a.itr_iters):
                if label == 'eager':
                    tr_e.train_iteration(itr, log=False)
                else:
                    step(itr)
                itr += 1
            torch.cuda.synchronize()
            res[label].append(1000.0 * (time.perf_counter() - t0) / a.itr_iters)
    for label, v in res.items():
        print("iteration %-6s ms: %s" % (label, " ".join("%.2f" % x for x in v)))


if __name__ == '__main__':
    main()
