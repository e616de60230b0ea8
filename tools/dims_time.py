"""What the zero-padded parameter layout costs: kernel times (CUDA events) of the policy gradient and Hessian-vector product at
M = 40 tasks, exact vs padded entry points at (2,2) N=2000 and (17,6) N=4000, padded only at (11,3) N=2000 (no exact kernel).
Each case times the per-task-parameter gradient (the inner SGD step of the meta-gradient chain) and the HVP at hidden 64,
with the default options (tensor cores on).  Writes one JSON line per case to stdout and, with --out FILE, to FILE.
usage: python tools/dims_time.py [--out FILE] [--iters N]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200 import _lib  # noqa: E402

CASES = [(2, 2, 2000, False), (2, 2, 2000, True), (17, 6, 4000, False), (17, 6, 4000, True), (11, 3, 2000, True)]


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def time_case(Do, Da, N, padded, iters, M=40, hidden=64):
    lib = _lib.load()
    suffix = '_padded' if padded else ''
    P = _lib.policy_layout(Do, Da, hidden)[3] if padded else lib.promp_num_params(Do, Da, hidden)
    dev = torch.device('cuda')
    g = torch.Generator(device='cuda').manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    theta = 0.1 * r(M, P)
    if padded:       # zero-pad invariant: only the logical entries are non-zero
        from promp_b200.policies.meta_gaussian_mlp_policy import MetaGaussianMLPPolicy
        pol = MetaGaussianMLPPolicy(name='t', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(hidden, hidden))
        keep = torch.zeros(P, dtype=torch.bool, device=dev)
        keep[pol._pad_index] = True
        theta *= keep
    obs, act, adv, mean, ls = r(M, N, Do), r(M, N, Da), r(M, N), r(M, N, Da), 0.1 * r(M, Da)
    grad, newp, out = (torch.empty(M, P, device=dev) for _ in range(3))
    vec = 0.01 * theta
    st = torch.zeros(M, 4, device=dev)
    need = getattr(lib, 'promp_policy_workspace_bytes' + suffix)(M, N, Do, Da, hidden)
    ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device=dev)
    s = _lib.stream()

    def grad_call():
        _lib.call('promp_policy_grad_ex' + suffix, Do, Da, hidden, M, N, None, _lib.ptr(theta), P, _lib.ptr(obs), _lib.ptr(act),
                  _lib.ptr(adv), _lib.ptr(mean), _lib.ptr(ls), 0, _lib.OBJ_RATIO, 1.0, 0.0, 0.0, 0, -13.8, _lib.ptr(grad),
                  _lib.ptr(newp), 0.1, _lib.ptr(st), None, None, None, None, _lib.ptr(ws), ws.numel() * 4, s)

    def hvp_call():
        _lib.call('promp_policy_hvp_ragged' + suffix, Do, Da, hidden, M, N, None, _lib.ptr(theta), P, _lib.ptr(obs), _lib.ptr(act),
                  _lib.ptr(adv), _lib.ptr(mean), _lib.ptr(ls), 0, _lib.OBJ_RATIO, 0.1, 5e-4, 0, -13.8, _lib.ptr(vec),
                  _lib.ptr(out), _lib.ptr(st), _lib.ptr(ws), ws.numel() * 4, s)

    def timeit(fn):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / iters * 1e3
    return dict(obs_dim=Do, act_dim=Da, N=N, M=M, hidden=hidden, entry='padded' if padded else 'exact', P=P,
                grad_us=round(timeit(grad_call), 1), hvp_us=round(timeit(hvp_call), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--iters', type=int, default=200)
    args = ap.parse_args()
    _lib.require_cuda()
    lines = [json.dumps(dict(gpu=gpu_info()))]
    for rep in range(2):          # two passes: the spread between them is the noise of the numbers
        for Do, Da, N, padded in CASES:
            res = time_case(Do, Da, N, padded, args.iters)
            res['pass'] = rep
            lines.append(json.dumps(res))
    for ln in lines:
        print(ln)
    if args.out:
        with open(args.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
