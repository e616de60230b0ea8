"""Run a fixed, seeded matrix of calls to the policy entry points of the library PROMP_B200_LIB selects and write every output
buffer to an .npz; or compare two such dumps byte for byte (uint8 views, so NaN payloads and untouched sentinel bytes
compare too).  A change to the policy kernels that must not change results leaves every array identical.

    PROMP_B200_LIB=path/to/lib.so python tools/policy_kernels_dump.py OUT.npz
    python tools/policy_kernels_dump.py --compare A.npz B.npz

The matrix: promp_policy_grad_ex, promp_policy_hvp_ragged, promp_policy_chain and promp_policy_forward with their *_padded
siblings, at the exact shapes (2,2), (4,2), (17,6) and the bucket shapes (1,1), (5,3), (11,3), (19,8), hidden 32 and 64,
tensor_cores 0 / 1 with tc_threads 256 / 512, chain 0 / 1 for a gradient-only and an HVP chain; geometries with one tile
per task, tasks split over several CTAs, CTAs spanning three or more tasks and N not a multiple of 64 / 128; param_stride
0 / P, n_valid NULL or ragged with poisoned (NaN) padding rows, ls_per_sample 0 / 1, a binding and a non-binding log_std
clip, every obj_kind with and without KL, grad / out_params / stats NULL or set, HVP out aliasing vec or not, a
device-resident KL multiplier, and the launch re-use producer with its consumer on a hit and on a miss.  Output buffers
start as NaN; the workspace's control words are recorded after every call (they must be left zero).
"""
import argparse
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200 import _lib  # noqa: E402

L = _lib
EXACT = ((2, 2), (4, 2), (17, 6))
BUCKETS = ((1, 1), (5, 3), (11, 3), (19, 8))
# (M, N): one tile per task; tasks split over several CTAs; CTAs spanning >= 3 tasks; N not a multiple of 64 / 128
GEOMS = ((3, 60), (2, 3001), (700, 50), (5, 777))
MODES = ((0, 0), (1, 256), (1, 512))       # (tensor_cores, tc_threads)


class Runner:
    def __init__(self):
        import torch
        self.torch = torch
        self.lib = L.load()
        self.stream = L.stream()
        self.out = {}
        self.data = {}

    def dev(self, a, dtype=None):
        return self.torch.as_tensor(np.ascontiguousarray(a), dtype=dtype or self.torch.float32, device='cuda')

    def nan(self, shape):
        return self.torch.full(shape, float('nan'), dtype=self.torch.float32, device='cuda')

    def check(self, rc, what):
        if rc != 0:
            raise RuntimeError('%s: rc %d: %s' % (what, rc, L.last_error()))

    def save(self, name, **bufs):
        self.torch.cuda.synchronize()
        for k, v in bufs.items():
            if v is not None:
                self.out['%s/%s' % (name, k)] = v.cpu().numpy()

    def layout(self, do, da, hidden, padded):
        if padded:
            return L.policy_layout(do, da, hidden)
        return do, da, hidden, self.lib.promp_num_params(do, da, hidden)

    def inputs(self, do, da, hidden, padded, M, N):
        """Seeded inputs of one (shape, hidden, geometry); every variant below reads these."""
        key = (do, da, hidden, padded, M, N)
        if key in self.data:
            return self.data[key]
        rng = np.random.default_rng([do, da, hidden, padded, M, N])
        _, dac, _, P = self.layout(do, da, hidden, padded)
        th = rng.normal(0, 0.3, (M, P)).astype(np.float32)
        th[:, P - dac:] = rng.uniform(-1.0, 0.3, (M, dac))          # log_std: some below the binding clip at -0.5
        nv = rng.integers(1, N + 1, M).astype(np.int32)
        nv[0] = N
        obs, act = rng.normal(0, 1, (M, N, do)), rng.normal(0, 1, (M, N, da))
        adv, mean = rng.normal(0, 1, (M, N)), rng.normal(0, 0.5, (M, N, da))
        ls_s, ls_t = rng.uniform(-1, 0.2, (M, N, da)), rng.uniform(-1, 0.2, (M, da))
        pad = np.arange(N)[None, :] >= nv[:, None]                  # ragged copies: poison the padding rows
        poison = lambda x: np.where(pad.reshape(pad.shape + (1,) * (x.ndim - 2)), np.nan, x)   # noqa: E731
        d = dict(P=P, th=self.dev(th), th0=self.dev(th[:1]), nv=self.dev(nv, self.torch.int32),
                 vec=self.dev(rng.normal(0, 0.05, (M, P))), klm=self.dev(np.array([1.5])))
        for tag, f in (('', lambda x: x), ('_r', poison)):
            d['obs' + tag], d['act' + tag], d['adv' + tag] = self.dev(f(obs)), self.dev(f(act)), self.dev(f(adv))
            d['mean' + tag], d['ls_s' + tag] = self.dev(f(mean)), self.dev(f(ls_s))
        d['ls_t'] = d['ls_t_r'] = self.dev(ls_t)
        self.data[key] = d
        return d

    def workspace(self, nbytes):
        return self.torch.zeros((nbytes + 3) // 4, dtype=self.torch.int32, device='cuda')

    def grad(self, tag, do, da, hidden, padded, M, N, stride, ragged, ls_ps, obj, kl, clip, want_grad, want_out, want_stats,
             reuse=None):
        d = self.inputs(do, da, hidden, padded, M, N)
        P, r = d['P'], '_r' if ragged else ''
        fn = getattr(self.lib, 'promp_policy_grad_ex_padded' if padded else 'promp_policy_grad_ex')
        wsb = getattr(self.lib, 'promp_policy_workspace_bytes_padded' if padded else 'promp_policy_workspace_bytes')(M, N, do, da,
                                                                                                                   hidden)
        ws = self.workspace(wsb)
        grad = self.nan((M, P)) if want_grad else None
        newp = self.nan((M, P)) if want_out else None
        st = self.nan((M, 4)) if want_stats else None
        flag = theta = unc = tcopy = None
        if reuse == 'produce':
            unc, tcopy = self.torch.full((1,), -7, dtype=self.torch.int32, device='cuda'), self.nan((P,))
        elif reuse in ('hit', 'miss'):
            flag = self.dev(np.array([1]), self.torch.int32)
            theta = d['th0'].clone().view(-1)
            if reuse == 'miss':
                theta[P // 2] += 1.0
        p = lambda x: x.data_ptr() if x is not None else None   # noqa: E731
        params = d['th0'] if stride == 0 else d['th']
        clip_on, min_ls = (1, -0.5) if clip == 'binding' else (0, -20.0)
        self.check(fn(do, da, hidden, M, N, p(d['nv']) if ragged else None, p(params), stride, p(d['obs' + r]), p(d['act' + r]),
                      p(d['adv' + r]), p(d['mean' + r]), p(d['ls_s' + r] if ls_ps else d['ls_t']), ls_ps, obj, 0.7, 0.2, kl,
                      clip_on, min_ls, p(grad), p(newp), 0.1, p(st), p(flag), p(theta), p(unc), p(tcopy), p(ws), ws.numel() * 4,
                      self.stream), tag)
        self.save(tag, grad=grad, out_params=newp, stats=st, unclipped=unc, theta_copy=tcopy, ctrl=ws[:M])

    def hvp(self, tag, do, da, hidden, padded, M, N, stride, ragged, ls_ps, obj, kl, clip, inplace):
        d = self.inputs(do, da, hidden, padded, M, N)
        P, r = d['P'], '_r' if ragged else ''
        fn = getattr(self.lib, 'promp_policy_hvp_ragged_padded' if padded else 'promp_policy_hvp_ragged')
        wsb = getattr(self.lib, 'promp_policy_workspace_bytes_padded' if padded else 'promp_policy_workspace_bytes')(M, N, do, da,
                                                                                                                   hidden)
        ws = self.workspace(wsb)
        vec = d['vec'].clone()
        out = vec if inplace else self.nan((M, P))
        st = self.nan((M, 4))
        p = lambda x: x.data_ptr() if x is not None else None   # noqa: E731
        clip_on, min_ls = (1, -0.5) if clip == 'binding' else (0, -20.0)
        self.check(fn(do, da, hidden, M, N, p(d['nv']) if ragged else None, p(d['th0'] if stride == 0 else d['th']), stride,
                      p(d['obs' + r]), p(d['act' + r]), p(d['adv' + r]), p(d['mean' + r]), p(d['ls_s' + r] if ls_ps else d['ls_t']),
                      ls_ps, obj, 0.1, kl, clip_on, min_ls, p(vec), p(out), p(st), p(ws), ws.numel() * 4, self.stream), tag)
        self.save(tag, out=out, stats=st, ctrl=ws[:M])

    def forward(self, tag, do, da, hidden, padded, M, N, stride):
        d = self.inputs(do, da, hidden, padded, M, N)
        mean = self.nan((M, N, da))
        fn = getattr(self.lib, 'promp_policy_forward_padded' if padded else 'promp_policy_forward')
        self.check(fn(do, da, hidden, M, N, (d['th0'] if stride == 0 else d['th']).data_ptr(), stride, d['obs'].data_ptr(),
                      mean.data_ptr(), self.stream), tag)
        self.save(tag, mean=mean)

    def chain(self, tag, do, da, hidden, padded, M, N, with_hvp, ragged, reuse):
        """Gradient chain: inner gradient + SGD step on shared parameters, outer gradient at the adapted ones; with_hvp adds
        two HVP stages v <- v - alpha H v + c grad KL (the second in place, with a device-resident KL multiplier)."""
        d = self.inputs(do, da, hidden, padded, M, N)
        P, r = d['P'], '_r' if ragged else ''
        p = lambda x: x.data_ptr() if x is not None else None   # noqa: E731
        th1, g0, g1, st = self.nan((M, P)), self.nan((M, P)), self.nan((M, P)), self.nan((4, M, 4))
        v1 = self.nan((M, P))
        common = dict(N=N, n_valid=p(d['nv']) if ragged else None, obs=p(d['obs' + r]), act=p(d['act' + r]), adv=p(d['adv' + r]),
                      old_mean=p(d['mean' + r]))
        stages = [dict(kind=0, params=p(d['th0']), param_stride=0, old_log_std=p(d['ls_t']), ls_per_sample=0, obj_kind=L.OBJ_LOGLIK,
                       obj_scale=1.0, kl_coeff=0.0, clip_log_std=1, grad=p(g0), out_params=p(th1), sgd_lr=0.1, stats=p(st[0])),
                  dict(kind=0, params=p(th1), param_stride=P, old_log_std=p(d['ls_s' + r]), ls_per_sample=1,
                       obj_kind=L.OBJ_CLIP, obj_scale=1.0, clip_eps=0.2, kl_coeff=0.05, clip_log_std=1, grad=p(g1),
                       stats=p(st[1]))]
        if with_hvp:
            stages += [dict(kind=1, params=p(d['th0']), param_stride=0, old_log_std=p(d['ls_t']), ls_per_sample=0,
                            obj_kind=L.OBJ_RATIO, kl_coeff=0.02, clip_log_std=1, inner_lr=0.1, vec=p(g1), out=p(v1), stats=p(st[2])),
                       dict(kind=1, params=p(d['th']), param_stride=P, old_log_std=p(d['ls_s' + r]), ls_per_sample=1,
                            obj_kind=L.OBJ_LOGLIK, kl_coeff=0.02, kl_coeff_dev=p(d['klm']), clip_log_std=1, inner_lr=0.1,
                            vec=p(v1), out=p(v1), stats=p(st[3]))]
        arr = (L.PolicyStage * len(stages))()
        for i, s in enumerate(stages):
            for k, v in {**common, **s}.items():
                setattr(arr[i], k, v)
        sfx = '_padded' if padded else ''
        nbytes = getattr(self.lib, 'promp_policy_chain_workspace_bytes' + sfx)(do, da, hidden, M, len(stages), ctypes.byref(arr))
        ws = self.workspace(nbytes)
        flag = theta = None
        if reuse in ('hit', 'miss'):
            flag = self.dev(np.array([1]), self.torch.int32)
            theta = d['th0'].clone().view(-1)
            if reuse == 'miss':
                theta[0] += 1.0
        self.check(getattr(self.lib, 'promp_policy_chain' + sfx)(do, da, hidden, M, -0.5, len(stages), ctypes.byref(arr), p(flag),
                                                                 p(theta), p(ws), ws.numel() * 4, self.stream), tag)
        ctrl = (4 + 12 * M + 31) // 32 * 32            # the chain's control words; one launch per stage: then their counters
        if getattr(self.lib, 'promp_policy_chain_num_launches' + sfx)(do, da, hidden, M, len(stages), ctypes.byref(arr)) > 1:
            ctrl += M
        self.save(tag, theta1=th1, grad0=g0, grad1=g1, stats=st, v1=v1 if with_hvp else None, ctrl=ws[:ctrl])


def dump(path):
    lib = L.load()
    r = Runner()
    n = 0
    for padded, shapes in ((False, EXACT), (True, BUCKETS)):
        for do, da in shapes:
            for hidden in (32, 64):
                for tc, tct in (MODES if hidden == 64 else MODES[:1]):
                    L.set_option('tensor_cores', tc)
                    L.set_option('tc_threads', tct)
                    base = 'p%d_o%d_a%d_h%d_tc%d_%d' % (padded, do, da, hidden, tc, tct)
                    sh = (do, da, hidden, padded)
                    for gi, (M, N) in enumerate(GEOMS):
                        g = '%s/g%d' % (base, gi)
                        P = r.inputs(*sh, M, N)['P']
                        for obj in (L.OBJ_RATIO, L.OBJ_LOGLIK, L.OBJ_CLIP, L.OBJ_NONE):
                            for kl in (0.0, 0.05):
                                r.grad('%s/grad_o%d_kl%g' % (g, obj, kl), *sh, M, N, 0 if obj % 2 else P, False, obj % 2,
                                       obj, kl, 'binding' if kl else 'free', True, True, True)
                        r.grad(g + '/grad_ragged_pertask', *sh, M, N, P, True, 1, L.OBJ_RATIO, 0.05,
                               'binding', True, False, True)
                        r.grad(g + '/grad_values_only', *sh, M, N, 0, True, 0, L.OBJ_CLIP, 0.05, 'free', False, False, True)
                        r.grad(g + '/grad_no_stats', *sh, M, N, 0, False, 1, L.OBJ_LOGLIK, 0.0, 'binding', True, False, False)
                        for obj in (L.OBJ_RATIO, L.OBJ_LOGLIK):
                            for ragged in (False, True):
                                r.hvp('%s/hvp_o%d_r%d' % (g, obj, ragged), *sh, M, N, 0 if ragged else P, ragged,
                                      int(ragged), obj, 0.02 * obj, 'binding' if ragged else 'free', inplace=obj == L.OBJ_LOGLIK)
                        r.forward(g + '/forward', *sh, M, N, 0 if gi % 2 else P)
                        n += 1
                    M, N = GEOMS[3]
                    for reuse in ('produce', 'hit', 'miss'):
                        r.grad('%s/reuse_%s' % (base, reuse), *sh, M, N, 0, False, 0, L.OBJ_LOGLIK, 0.0, 'binding', True, True, True,
                               reuse=reuse)
                    for chain in (0, 1):
                        L.set_option('chain', chain)
                        for gi, (M, N) in enumerate(GEOMS):
                            for with_hvp in (False, True):
                                r.chain('%s/chain%d_g%d_hvp%d' % (base, chain, gi, with_hvp), *sh, M, N, with_hvp, gi % 2 == 1, None)
                        for reuse in ('hit', 'miss'):
                            r.chain('%s/chain%d_reuse_%s' % (base, chain, reuse), *sh, *GEOMS[3], True, False, reuse)
                    L.set_option('chain', -1)
    L.set_option('tensor_cores', 1)
    L.set_option('tc_threads', 0)
    out = r.out
    ctrl = [k for k in out if k.endswith('/ctrl')]
    nonzero = [k for k in ctrl if np.any(out[k] != 0)]
    np.savez(path, **out)
    print('%s: %d arrays, %d bytes from %s; %d workspaces, %d with non-zero control words%s' % (
        path, len(out), sum(v.nbytes for v in out.values()), L.LIB_PATH, len(ctrl), len(nonzero),
        ''.join('\n  ' + k for k in nonzero[:20])))
    return 1 if nonzero else 0


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        x, y = a[k], b[k]
        if x.dtype != y.dtype or x.shape != y.shape or not np.array_equal(x.view(np.uint8), y.view(np.uint8)):
            bad.append(k)
    print('%d arrays compared, %d differ%s' % (len(set(a.files) | set(b.files)), len(bad), ''.join('\n  ' + k for k in bad[:50])))
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out', nargs='?')
    ap.add_argument('--compare', nargs=2, metavar=('A', 'B'))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    sys.exit(dump(args.out))


if __name__ == '__main__':
    main()
