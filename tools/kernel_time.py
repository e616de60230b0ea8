"""Time promp_policy_grad / promp_policy_hvp in isolation on synthetic data (CUDA events, L2-warm like the real loop).
usage: PROMP_B200_LIB=/path/to/variant.so python tools/kernel_time.py [point|cheetah] [64|32]   (hidden size; 32 runs the
CUDA-core kernels)"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200 import _lib  # noqa: E402


def main():
    wl = sys.argv[1] if len(sys.argv) > 1 else 'point'
    hid = int(sys.argv[2]) if len(sys.argv) > 2 else 64
    if os.environ.get('PROMP_TC'):
        _lib.set_option('tensor_cores', int(os.environ['PROMP_TC']))
    if os.environ.get('PROMP_TC_THREADS'):
        _lib.set_option('tc_threads', int(os.environ['PROMP_TC_THREADS']))
    Do, Da, M, N = (2, 2, 40, 2000) if wl == 'point' else (17, 6, 40, 4000)
    P = _lib.load().promp_num_params(Do, Da, hid)
    dev = torch.device('cuda')
    g = torch.Generator(device='cuda').manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    theta = 0.1 * r(P)
    theta_t = theta.view(1, -1).repeat(M, 1).contiguous()
    obs, act, adv, mean, ls = r(M, N, Do), r(M, N, Da), r(M, N), r(M, N, Da), 0.1 * r(M, Da)
    grad, newp, vec, out = torch.empty(M, P, device=dev), torch.empty(M, P, device=dev), 0.01 * r(M, P), torch.empty(M, P, device=dev)
    st = torch.zeros(M, 4, device=dev)
    need = _lib.load().promp_policy_workspace_bytes(M, N, Do, Da, hid)
    ws = torch.zeros((need + 3) // 4, dtype=torch.int32, device=dev)
    s = _lib.stream()

    def grad_call(stride, eval_only=False):
        _lib.call('promp_policy_grad', Do, Da, hid, M, N, _lib.ptr(theta if stride == 0 else theta_t), stride, _lib.ptr(obs),
                  _lib.ptr(act), _lib.ptr(adv), _lib.ptr(mean), _lib.ptr(ls), 0, 0, 1.0, 0.3, 0.0, 0, -13.8,
                  None if eval_only else _lib.ptr(grad), None if eval_only else _lib.ptr(newp), 0.1, _lib.ptr(st), _lib.ptr(ws),
                  ws.numel() * 4, s)

    def hvp_call(stride):
        _lib.call('promp_policy_hvp', Do, Da, hid, M, N, _lib.ptr(theta if stride == 0 else theta_t), stride, _lib.ptr(obs),
                  _lib.ptr(act), _lib.ptr(adv), _lib.ptr(mean), _lib.ptr(ls), 0, 0, 0.1, 5e-4, 0, -13.8, _lib.ptr(vec),
                  _lib.ptr(out), _lib.ptr(st), _lib.ptr(ws), ws.numel() * 4, s)

    def timeit(fn, n=30):
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

    print('%s hidden %d lib=%s' % (wl, hid, os.path.basename(_lib.LIB_PATH)))
    print('  grad shared-theta  %.1f us' % timeit(lambda: grad_call(0)))
    print('  grad per-task      %.1f us' % timeit(lambda: grad_call(P)))
    print('  grad eval-only     %.1f us' % timeit(lambda: grad_call(P, True)))
    print('  hvp  shared-theta  %.1f us' % timeit(lambda: hvp_call(0)))
    print('  hvp  per-task      %.1f us' % timeit(lambda: hvp_call(P)))
    lib = _lib.load()
    if hasattr(lib, 'promp_debug_phase_clocks'):          # -DPROMP_EXP_CLOCKS experiment build only
        import ctypes
        buf = (ctypes.c_ulonglong * 16)()
        lib.promp_debug_phase_clocks(buf, 1)
        n = 20
        for _ in range(n):
            grad_call(P)
        lib.promp_debug_phase_clocks(buf, 1)
        names = ['load X', 'layer0 (SIMT)', 'fwd MMA (sync+issue+wait)', 'tanh/MUP/A1 + sync', 'head + sync', 'gW2 col role + sync',
                 'D2 + fences + sync', 'wgrad SIMT (overlaps bwd MMA)', 'bwd MMA wait + ld + sync', 'D1 + sync', 'gW0 col role',
                 'flush: return', 'load_task', 'fwd MMA sync+issue (part of fwd MMA)', 'flush: W1 / b partials',
                 'flush: W0 / W2 partials, ticket, last arriver']
        tot = sum(buf[i] for i in range(16))
        print('  CTA 0 phase clocks per launch (grad per-task), total %.0f clk:' % (tot / n))
        for i, nm in enumerate(names):
            print('    %-34s %8.0f clk  %5.1f %%' % (nm, buf[i] / n, 100.0 * buf[i] / max(tot, 1)))


if __name__ == '__main__':
    main()
