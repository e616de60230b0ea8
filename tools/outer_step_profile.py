"""Where the ProMP outer step's time goes between its launches: one torch.profiler trace (CUDA activities) of a few replays of
the benchmark's captured meta-iteration, and a tiles-per-CTA sweep of the stand-alone gradient / HVP kernels.

usage: python tools/outer_step_profile.py [point|cheetah] [--out DIR] [--replays R]

Writes trace_<workload>.json (chrome trace) and summary_<workload>.txt / .json into DIR (default outer_step_profile_out/),
and prints the summary:
  - the iteration time (CUDA events, profiler off) of the benchmark's step() and of the bare graph replay without step()'s
    host part (the task draw and its upload), alternated three times;
  - the sum of kernel durations of one replay against its first-to-last span: the difference is the inter-kernel gaps;
  - every launch of the outer step (the K Adam epochs and the statistics pass, i.e. everything after the second sampling
    phase's processing kernel) with its duration and the gap before it;
  - each policy kernel's duration at 1..5 tiles per CTA (M = 40, N = 128 k), fitted as a + b * q: `a` is the part of a launch
    that does not scale with its tiles (ramp-up, weight staging, flush and last-arriver drain), an upper bound on what
    removing a launch boundary can save inside the kernel; the in-graph duration less q * b is the same quantity measured in
    place."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from promp_b200 import _lib  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ', power limit not read'
    return q


def kernels_of(prof):
    """(name, start us, duration us) of every device kernel, in start order."""
    out = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith('Memcpy'):
            out.append((e.name, e.time_range.start, e.time_range.end - e.time_range.start))
    out.sort(key=lambda x: x[1])
    return out


def short(name):
    n = name.split('(')[0].split('<')[0]
    return n.replace('void ', '').strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('workload', nargs='?', default='point', choices=['point', 'cheetah'])
    ap.add_argument('--out', default='outer_step_profile_out')
    ap.add_argument('--replays', type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import bench
    from promp_b200.utils import logger
    logger.set_quiet(True)
    _lib.require_cuda()
    lines = []

    def say(s=''):
        print(s)
        lines.append(s)
    say('card: ' + card())
    wl = bench.WORKLOADS[args.workload]
    np.random.seed(1)
    tr = bench.build_stack(wl, 'device')
    step = tr.capture_graph(warmup=2)
    graph = tr._graph

    def time_us(fn, n=200):
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n * 1e3
    t_step, t_bare = [], []
    for _ in range(3):
        t_step.append(time_us(step))
        t_bare.append(time_us(graph.replay))
    replay_us = float(np.median(t_step))
    say('%s: us per iteration, step() %s, bare graph replay %s: step()\'s host part leaves the device idle %.1f us '
        '(%.1f %%)' % (args.workload, ' '.join('%.1f' % t for t in t_step), ' '.join('%.1f' % t for t in t_bare),
                       replay_us - np.median(t_bare), 100.0 * (replay_us - np.median(t_bare)) / replay_us))

    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.replays):
            step()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(args.out, 'trace_%s.json' % args.workload))
    ks = kernels_of(prof)
    per = len(ks) // args.replays
    assert per * args.replays == len(ks), "kernels per replay differ: %d over %d replays" % (len(ks), args.replays)
    reps = [ks[i * per:(i + 1) * per] for i in range(args.replays)]
    busy = np.array([sum(d for _, _, d in r) for r in reps])
    span = np.array([r[-1][1] + r[-1][2] - r[0][1] for r in reps])
    say('%d kernels per replay; kernel sum %.1f us, first-to-last span %.1f us, gaps inside the span %.1f us (profiled, '
        'median over %d replays of step())' % (per, np.median(busy), np.median(span), np.median(span - busy), args.replays))
    # the outer step: everything after the second processing kernel
    names = [short(k[0]) for k in reps[0]]
    proc = [i for i, nm in enumerate(names) if 'process' in nm]
    first = proc[1] + 1 if len(proc) >= 2 else 0
    say('outer step: launches %d..%d of the replay (%d launches)' % (first, per - 1, per - first))
    say('  %-4s %-34s %9s %9s' % ('#', 'kernel', 'dur us', 'gap us'))
    dur = np.median(np.array([[k[2] for k in r] for r in reps]), axis=0)
    gap = np.median(np.array([[0.0] + [r[i][1] - (r[i - 1][1] + r[i - 1][2]) for i in range(1, per)] for r in reps]), axis=0)
    for i in range(first, per):
        say('  %-4d %-34s %9.1f %9.1f' % (i, names[i][:34], dur[i], gap[i]))
    outer_busy, outer_gap = float(dur[first:].sum()), float(gap[first:].sum())
    say('  outer step: kernels %.1f us, gaps %.1f us (%.1f %% of the iteration)' %
        (outer_busy, outer_gap, 100.0 * outer_gap / replay_us))

    # stand-alone tiles-per-CTA sweep
    Do, Da = wl['Do'], wl['Da']
    M, P = wl['M'], _lib.load().promp_num_params(Do, Da, 64)
    dev = torch.device('cuda')
    g = torch.Generator(device='cuda').manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    theta = 0.1 * r(P)
    theta_t = theta.view(1, -1).repeat(M, 1).contiguous()
    s = _lib.stream()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fits = {}
    say('stand-alone kernels (M = %d, per-task parameters), us per launch by tiles per CTA q:' % M)
    for kind in ('grad', 'hvp'):
        pts = []
        for k in sorted({max(1, (q * sms) // M) for q in (1, 2, 3, 4, 5)}):
            N = 128 * k
            T = M * k
            q = -(-T // min(T, sms))
            obs, act, adv, mean, ls = r(M, N, Do), r(M, N, Da), r(M, N), r(M, N, Da), 0.1 * r(M, Da)
            grad, vec, out = torch.empty(M, P, device=dev), 0.01 * r(M, P), torch.empty(M, P, device=dev)
            st = torch.zeros(M, 4, device=dev)
            need = _lib.load().promp_policy_workspace_bytes(M, N, Do, Da, 64)
            ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device=dev)
            if kind == 'grad':
                fn = lambda: _lib.call('promp_policy_grad', Do, Da, 64, M, N, _lib.ptr(theta_t), P, _lib.ptr(obs), _lib.ptr(act),
                                       _lib.ptr(adv), _lib.ptr(mean), _lib.ptr(ls), 0, 0, 1.0, 0.3, 0.0, 0, -13.8, _lib.ptr(grad),
                                       None, 0.1, _lib.ptr(st), _lib.ptr(ws), ws.numel() * 4, s)
            else:
                fn = lambda: _lib.call('promp_policy_hvp', Do, Da, 64, M, N, _lib.ptr(theta_t), P, _lib.ptr(obs), _lib.ptr(act),
                                       _lib.ptr(adv), _lib.ptr(mean), _lib.ptr(ls), 0, 0, 0.1, 5e-4, 0, -13.8, _lib.ptr(vec),
                                       _lib.ptr(out), _lib.ptr(st), _lib.ptr(ws), ws.numel() * 4, s)
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as p2:
                for _ in range(30):
                    fn()
                torch.cuda.synchronize()
            d = float(np.median([k_[2] for k_ in kernels_of(p2)]))
            pts.append((q, d))
            say('  %-4s N = %5d  q = %d  %7.1f us' % (kind, N, q, d))
            del obs, act, adv, mean, ls, grad, vec, out, ws
        qq, dd = np.array([p_[0] for p_ in pts], float), np.array([p_[1] for p_ in pts])
        slope, icpt = np.polyfit(qq, dd, 1)
        fits[kind] = (icpt, slope)
        say('  %-4s fit: %.1f us + %.1f us per tile per CTA' % (kind, icpt, slope))
    # in-graph fixed part of each outer-step policy launch
    T = M * -(-(wl['E'] * wl['H']) // 128)
    q_b = -(-T // min(T, sms))
    fixed = 0.0
    nfix = 0
    for i in range(first, per):
        kind = 'hvp' if 'hvp' in names[i] else ('grad' if 'grad' in names[i] else None)
        if kind is None or dur[i] < 0.5 * fits[kind][1] * q_b:     # the skipped epoch-1 inner gradient exits at once
            continue
        fixed += dur[i] - q_b * fits[kind][1]
        nfix += 1
    say('in-graph fixed part of the %d outer-step policy launches at q = %d: %.1f us (%.1f %% of the iteration); with the gaps '
        '%.1f us (%.1f %%)' % (nfix, q_b, fixed, 100.0 * fixed / replay_us, fixed + outer_gap,
                               100.0 * (fixed + outer_gap) / replay_us))
    with open(os.path.join(args.out, 'summary_%s.txt' % args.workload), 'w') as f:
        f.write('\n'.join(lines) + '\n')
    with open(os.path.join(args.out, 'summary_%s.json' % args.workload), 'w') as f:
        json.dump(dict(step_us=t_step, bare_replay_us=t_bare, kernels=[(names[i], float(dur[i]), float(gap[i])) for i in range(per)],
                       fits=fits, outer_first=first), f, indent=1)


if __name__ == '__main__':
    main()
