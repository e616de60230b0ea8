"""The work-item plans of the dataflow chain kernel (policy_chain_tc_kernel, DESIGN.md section 3.7) and the meta-gradient it
computes under each of them, against float64.

plan_chain (csrc/policy.cu) splits every stage of a chain into items of q consecutive 128-sample tiles of one task; the last
stage tapers to q/2 and then 1 tile per item over up to three task regions.  The kernel decodes an item id back into
(stage, region, task, tiles) and spins on per-task ready flags, so a plan or decode error gives wrong gradients for some
tasks only, or a hang.

CPU tests: a Python copy of plan_chain against promp_policy_chain_plan_info field by field over a sweep of task counts,
sample counts, stage lists and the chain_q / chain_taper options; the plan invariants, with every item decoded the way the
kernel decodes it; the plans of the GPU cases pinned at 132 SMs (H100 SXM); and the split of chains longer than six stages
(three or more inner steps) into consecutive launches.

GPU tests (-m gpu): ProMP and TRPO-MAML meta-gradient evaluations (_objective_pass / _meta_pass with reduce=False) under
every plan shape, per task and per parameter block against the float64 gradient of oracle/tf_half.meta_objective at the
bar of test_policy_oracle.py, with pad entries exactly 0, the stats rows checked, run-to-run bit identity and the control
words left zero; then every case again in reverse order on one shared workspace, bit-identical to the first pass.
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

import test_policy_oracle as po
from oracle import tf_half as th

TBT = 128                 # samples per tile of the tensor-core kernels
MAX_STAGES = 6            # CHAIN_MAX_STAGES
PSTAT = 4                 # stats floats per partial slot
SXM_SMS = 132             # H100 SXM
FIELDS = 15               # ints per stage in promp_policy_chain_plan_info's output


def ctrl_bytes(M):
    """chain_ctrl_bytes (csrc/policy.cu): queue words, the dataflow kernel's ready flags and arrival counters, then the
    one-launch-per-stage path's arrival counters, 128-byte aligned."""
    return -(-(16 + 2 * MAX_STAGES * M * 4 + -(-M * 4 // 16) * 16) // 128) * 128


# ------------------------------------------------------------------------------------------------------ the plan copy
def plan_chain(Ns, M, sms=SXM_SMS, chain_q=0, taper=1, kinds=None):
    """Python copy of plan_chain (csrc/policy.cu): [sms, n_items] + 15 ints per stage, the layout of
    promp_policy_chain_plan_info: ntiles, item_base, n_items, n_regions, reg_m0[4], reg_q[3], reg_item0[3], kind."""
    kinds = kinds or [0] * len(Ns)
    out, base = [sms, 0], 0
    for s, N in enumerate(Ns):
        ntiles = -(-N // TBT)
        q = 4
        if chain_q > 0:
            q = chain_q
        else:
            while q > 1 and M * -(-ntiles // q) < sms:
                q >>= 1
        q = min(q, ntiles)
        if taper and s == len(Ns) - 1 and q > 1 and M >= 4:
            q2 = q // 2 if q > 2 else q
            mB = M - M // 4
            mA = M // 2 if q2 < q else mB
            m0, qs = (0, mA, mB, M), (q, q2, 1)
            regions = [(m0[r], m0[r + 1], qs[r]) for r in range(3) if m0[r + 1] > m0[r]]
        else:
            regions = [(0, M, q)]
        reg_m0, reg_q, reg_item0 = [0] * 4, [0] * 3, [0] * 3
        items = 0
        for r, (a, b, qr) in enumerate(regions):
            reg_m0[r], reg_q[r], reg_item0[r] = a, qr, items
            items += (b - a) * -(-ntiles // qr)
        reg_m0[len(regions)] = M
        out += [ntiles, base, items, len(regions)] + reg_m0 + reg_q + reg_item0 + [kinds[s]]
        base += items
    out[1] = base
    return out


def stage_fields(plan, s):
    o = plan[2 + FIELDS * s: 2 + FIELDS * (s + 1)]
    return dict(ntiles=o[0], item_base=o[1], n_items=o[2], n_regions=o[3], reg_m0=o[4:8], reg_q=o[8:11], reg_item0=o[11:14])


def regions_of(plan, n_stages):
    """[(ntiles, n_items, ((m0, m1, q), ...)) per stage]: the form the WANT_PLAN pins take."""
    out = []
    for s in range(n_stages):
        f = stage_fields(plan, s)
        regs = tuple((f['reg_m0'][r], f['reg_m0'][r + 1], f['reg_q'][r]) for r in range(f['n_regions']))
        out.append((f['ntiles'], f['n_items'], regs))
    return out


def _stages(kinds, Ns):
    from promp_b200 import _lib
    st = (_lib.PolicyStage * len(Ns))()
    for s, (k, N) in enumerate(zip(kinds, Ns)):
        st[s].kind, st[s].N = k, N
    return st


def plan_info(Ns, M, kinds=None):
    """promp_policy_chain_plan_info under the options currently set."""
    from promp_b200 import _lib
    kinds = kinds or [0] * len(Ns)
    out = (ctypes.c_int32 * (2 + FIELDS * len(Ns)))()
    rc = _lib.load().promp_policy_chain_plan_info(M, len(Ns), ctypes.cast(_stages(kinds, Ns), ctypes.c_void_p),
                                                  ctypes.cast(out, ctypes.c_void_p))
    assert rc == 0, _lib.last_error()
    return list(out)


@contextlib.contextmanager
def chain_options(chain=-1, chain_q=0, taper=1):
    from promp_b200 import _lib
    try:
        _lib.set_option('chain', chain)
        _lib.set_option('chain_q', chain_q)
        _lib.set_option('chain_taper', taper)
        yield
    finally:
        _lib.set_option('chain', -1)
        _lib.set_option('chain_q', 0)
        _lib.set_option('chain_taper', 1)


def check_invariants(plan, Ns, M):
    """Regions partition [0, M) in order; item_base is contiguous; decoding every item id as the kernel does
    (policy_chain_tc_kernel) covers each (stage, task)'s tiles exactly once, in order, with only the last item of a task short,
    and first_item / per_task name the task's own contiguous run of items."""
    n_stages = len(Ns)
    bases = np.array([stage_fields(plan, s)['item_base'] for s in range(n_stages)])
    base = 0
    for s in range(n_stages):
        f = stage_fields(plan, s)
        assert f['item_base'] == base, (s, f)
        assert f['ntiles'] == -(-Ns[s] // TBT)
        nr = f['n_regions']
        assert 1 <= nr <= 3
        m0 = f['reg_m0'][:nr + 1]
        assert m0[0] == 0 and m0[-1] == M and all(a < b for a, b in zip(m0[:-1], m0[1:])), (s, f)
        base += f['n_items']
    assert plan[1] == base
    it = np.arange(plan[1])
    st = np.searchsorted(bases, it, side='right') - 1     # the kernel's stage walk: last stage whose item_base <= it
    for s in range(n_stages):
        f = stage_fields(plan, s)
        nr, ntiles = f['n_regions'], f['ntiles']
        j = it[st == s] - f['item_base']
        assert len(j) == f['n_items']
        r = np.searchsorted(np.array(f['reg_item0'][:nr]), j, side='right') - 1
        q = np.array(f['reg_q'][:nr])[r]
        per_task = -(-ntiles // q)
        jr = j - np.array(f['reg_item0'][:nr])[r]
        mr, k = jr // per_task, jr % per_task
        m = np.array(f['reg_m0'][:nr])[r] + mr
        assert np.all(m < np.array(f['reg_m0'][1:nr + 1])[r]), 'item decoded into the next region'
        g_lo = m * ntiles + k * q
        g_hi = m * ntiles + np.minimum(k * q + q, ntiles)
        first = f['item_base'] + np.array(f['reg_item0'][:nr])[r] + mr * per_task
        glob = j + f['item_base']
        assert np.all((first <= glob) & (glob < first + per_task))
        assert np.all((g_hi - g_lo == q) | (k == per_task - 1)), 'only the last item of a task may be short'
        assert np.all(g_hi > g_lo)
        # items of a task in id order tile [m * ntiles, (m + 1) * ntiles) exactly once
        order = np.lexsort((g_lo, m))
        ms, lo, hi = m[order], g_lo[order], g_hi[order]
        assert np.array_equal(np.unique(ms), np.arange(M))
        start = np.r_[True, ms[1:] != ms[:-1]]
        end = np.r_[ms[1:] != ms[:-1], True]
        assert np.all(lo[start] == ms[start] * ntiles)
        assert np.all(hi[end] == (ms[end] + 1) * ntiles)
        assert np.all(lo[~start] == hi[np.flatnonzero(~start) - 1])


# ------------------------------------------------------------------------------------------------------------ CPU
SWEEP_M = (1, 2, 3, 4, 5, 7, 8, 10, 20, 40, 133, 140, 300)
SWEEP_N = (1, 128, 129, 391, 700, 830, 1000, 2000, 4000, 40000)
SWEEP_Q = (0, 1, 2, 3, 4, 5, 8, 64)


def _stage_lists(M):
    """Uniform lists of 1 to 6 stages at every sweep N, and ragged ones (a different N per stage)."""
    lists = [[N] * n for N in SWEEP_N for n in range(1, MAX_STAGES + 1)]
    rng = np.random.RandomState(M)
    for n in range(2, MAX_STAGES + 1):
        for _ in range(3):
            lists.append([int(x) for x in rng.choice(SWEEP_N, n)])
    lists += [[2000, 1800, 2000], [129, 40000, 1], [391, 700, 830, 1000, 128, 4000]]
    return lists


@pytest.mark.parametrize('taper', [1, 0])
@pytest.mark.parametrize('chain_q', SWEEP_Q)
def test_plan_info_matches_python_copy(chain_q, taper):
    from promp_b200 import _lib
    lib = _lib.load()
    with chain_options(chain_q=chain_q, taper=taper):
        for M in SWEEP_M:
            for Ns in _stage_lists(M):
                kinds = [0] * ((len(Ns) + 1) // 2) + [1] * (len(Ns) // 2)
                got = plan_info(Ns, M, kinds)
                want = plan_chain(Ns, M, sms=got[0], chain_q=chain_q, taper=taper, kinds=kinds)
                assert got == want, (M, Ns, chain_q, taper, got, want)
                check_invariants(got, Ns, M)
                st = _stages(kinds, Ns)
                ws = lib.promp_policy_chain_workspace_bytes(2, 2, 64, M, len(Ns), ctypes.cast(st, ctypes.c_void_p))
                assert ws >= ctrl_bytes(M) + got[1] * (4484 + PSTAT) * 4, (M, Ns, ws)


def test_plan_info_rejects_bad_arguments():
    from promp_b200 import _lib
    lib = _lib.load()
    out = (ctypes.c_int32 * (2 + FIELDS * 7))()
    st = _stages([0] * 7, [2000] * 7)
    p = lambda a: ctypes.cast(a, ctypes.c_void_p)
    for M, n in ((20, 7), (20, 0), (0, 3)):
        assert lib.promp_policy_chain_plan_info(M, n, p(st), p(out)) != 0
        assert 'promp_policy_chain_plan_info' in _lib.last_error()
    assert lib.promp_policy_chain_plan_info(20, 3, None, p(out)) != 0
    assert lib.promp_policy_chain_plan_info(20, 3, p(st), None) != 0
    # the size queries' -1 says why
    assert lib.promp_policy_chain_workspace_bytes(2, 2, 64, 20, 7, p(st)) == -1
    assert '1..6 stages' in _lib.last_error() and 'workspace_bytes' in _lib.last_error()
    assert lib.promp_policy_chain_num_launches(2, 2, 64, 0, 3, p(st)) == -1
    assert 'M=0' in _lib.last_error() and 'num_launches' in _lib.last_error()


def chain_kinds(S1, want_grad=True, explore=False):
    """Stage kinds and phase indices of MAMLAlgo._meta_pass's chain: inner steps, outer step, HVPs back to step 0, the
    exploration stage last."""
    kinds, ph = [0] * (S1 + 1), list(range(S1 + 1))
    if want_grad:
        kinds += [1] * S1
        ph += list(range(S1 - 1, -1, -1))
    if explore:
        kinds.append(0)
        ph.append(0)
    return kinds, ph


def pieces_of(kinds, Ns):
    return [(kinds[i:i + MAX_STAGES], Ns[i:i + MAX_STAGES]) for i in range(0, len(kinds), MAX_STAGES)]


# Plans at 132 SMs (H100 SXM) of the GPU cases: per launch, per stage (ntiles, n_items, ((m0, m1, q) per region)).  The
# last stage of every launch tapers.
_Q2_16 = (16, 160, ((0, 20, 2),))                       # M=20, N=2000: q = 2 (q = 4 would give 80 items < 132)
_TAPER_20 = (16, 200, ((0, 15, 2), (15, 20, 1)))         # q = 2 taper: q/2 = q, so the middle region is empty
WANT_PLAN = {
    'c1': [[_Q2_16, _Q2_16, _TAPER_20]],
    'c2': [[(32, 160, ((0, 10, 2),)), (32, 160, ((0, 10, 2),)), (32, 192, ((0, 8, 2), (8, 10, 1)))]],
    'c3': [[(16, 160, ((0, 10, 1),))] * 3],             # q = 1: no taper
    'c4': [[(16, 160, ((0, 40, 4),))] * 2 + [(16, 320, ((0, 20, 4), (20, 30, 2), (30, 40, 1)))]],
    'c4-notaper': [[(16, 160, ((0, 40, 4),))] * 3],
    'c5-700': [[(6, 14, ((0, 7, 3),))] * 2 + [(6, 30, ((0, 3, 3), (3, 6, 1), (6, 7, 1)))]],     # q/2 = 1: two q = 1 regions
    'c5-830': [[(7, 21, ((0, 7, 3),))] * 2 + [(7, 37, ((0, 3, 3), (3, 6, 1), (6, 7, 1)))]],     # 7 tiles: short last items
    'c6-M4': [[(8, 8, ((0, 4, 4),))] * 2 + [(8, 16, ((0, 2, 4), (2, 3, 2), (3, 4, 1)))]],
    'c6-M5': [[(8, 10, ((0, 5, 4),))] * 2 + [(8, 20, ((0, 2, 4), (2, 4, 2), (4, 5, 1)))]],
    'c7': [[(4, 5, ((0, 5, 4),))] * 2 + [(4, 10, ((0, 2, 4), (2, 4, 2), (4, 5, 1)))]],           # chain_q 64 clamped to 4
    'c8-140x100': [[(1, 140, ((0, 140, 1),))] * 3],
    'c8-1x40000': [[(313, 157, ((0, 1, 2),))] * 3],     # M < 4: no taper
    'c9-s2': [[_Q2_16] * 4 + [_TAPER_20]],
    'c9-explore-s2': [[_Q2_16] * 5 + [_TAPER_20]],
    'c10-s0': [[_TAPER_20]],
    'c10-s3': [[_Q2_16] * 5 + [_TAPER_20], [_TAPER_20]],
    'c10-s4': [[_Q2_16] * 5 + [_TAPER_20], [_Q2_16, _Q2_16, _TAPER_20]],
    'c11-ragged': [[_Q2_16, (15, 160, ((0, 20, 2),)), _TAPER_20]],
    'c14-s3-mixed': [[(8, 160, ((0, 20, 1),))] * 3 + [(6, 120, ((0, 20, 1),))] + [(8, 160, ((0, 20, 1),))] * 2,
                     [(8, 160, ((0, 20, 1),))]],      # q = 1 throughout: no taper
}


class ChainCase(object):
    """One meta-gradient evaluation: shape, algorithm, inner steps, phase sizes, chain options."""

    def __init__(self, cid, Do=2, Da=2, M=20, N=2000, S1=1, algo='promp', chain=-1, chain_q=0, taper=1, explore=False,
                 act='tanh', out_tanh=False, n_valid=None, Ns=None, reuse=False, plan=None, launches=None):
        self.plan = plan or cid          # its WANT_PLAN entry
        self.launches = launches         # kernels launched per piece (None: one dataflow launch each)
        self.cid, self.Do, self.Da, self.M, self.S1 = cid, Do, Da, M, S1
        self.algo, self.chain, self.chain_q, self.taper, self.explore = algo, chain, chain_q, taper, explore
        self.act, self.out_tanh, self.reuse = act, out_tanh, reuse
        self.n_valid = n_valid          # per phase: per-task valid counts (RaggedPhaseData) or None
        self.Ns = list(Ns) if Ns is not None else [N] * (S1 + 1)

    def __repr__(self):
        return self.cid

    def stage_Ns(self):
        kinds, ph = chain_kinds(self.S1, explore=self.explore)
        return kinds, [self.phase_N(p) for p in ph]

    def phase_N(self, s):
        if self.n_valid is not None and self.n_valid[s] is not None:
            return (max(self.n_valid[s]) + 3) // 4 * 4          # RaggedPhaseData's row stride
        return self.Ns[s]


RAGGED_NV = [[1, 128, 129] + [2000 - 37 * i for i in range(17)],
             [129, 1, 128] + [1800 - 41 * i for i in range(17)]]

MIXED_NV = [[1, 128, 129] + [top - 23 * i for i in range(17)] for top in (1024, 1000, 900, 700)]

CASES = [
    ChainCase('c1'),
    ChainCase('c1-trpo', algo='trpo', plan='c1'),
    ChainCase('c2', Do=17, Da=6, M=10, N=4000),
    ChainCase('c3', M=10),
    ChainCase('c4', M=40, chain=1),
    ChainCase('c4-notaper', M=40, chain=1, taper=0),
    ChainCase('c5-700', M=7, N=700, chain=1, chain_q=3),
    ChainCase('c5-830', M=7, N=830, chain=1, chain_q=3),
    ChainCase('c6-M4', Do=4, M=4, N=1000, chain=1, chain_q=4),
    ChainCase('c6-M5', Do=4, M=5, N=1000, chain=1, chain_q=4),
    ChainCase('c7', M=5, N=391, chain=1, chain_q=64),
    ChainCase('c7-5x3', Do=5, Da=3, M=5, N=391, chain=1, chain_q=64, plan='c7'),
    ChainCase('c8-140x100', M=140, N=100),
    ChainCase('c8-1x40000', M=1, N=40000),
    ChainCase('c9-s2', S1=2),
    ChainCase('c9-trpo-explore-s2', S1=2, algo='trpo', explore=True, plan='c9-explore-s2'),
    ChainCase('c10-s0', S1=0),
    ChainCase('c10-s0-trpo', S1=0, algo='trpo', plan='c10-s0'),
    ChainCase('c10-s3', S1=3),
    ChainCase('c10-s3-trpo', S1=3, algo='trpo', plan='c10-s3'),
    ChainCase('c10-s4', S1=4),
    ChainCase('c10-s4-trpo', S1=4, algo='trpo', plan='c10-s4'),
    ChainCase('c11-ragged', n_valid=RAGGED_NV),
    ChainCase('c12-relu', act='relu', plan='c1'),
    ChainCase('c12-otanh', out_tanh=True, plan='c1'),
    ChainCase('c12-relu-otanh', act='relu', out_tanh=True, plan='c1'),
    ChainCase('c13-reuse', reuse=True, plan='c1'),
    # three inner steps on ragged phases whose pieces take different paths on one workspace: piece 1 holds the outer step on
    # phase 3 (6 tiles, 120 < 132 tiles in all: one launch per stage), piece 2 the HVP on phase 0 (8 tiles: dataflow)
    ChainCase('c14-s3-mixed', S1=3, n_valid=MIXED_NV, launches=[6, 1]),
]


def test_want_plan_pins_match_the_python_copy_at_132_sms():
    for case in CASES:
        kinds, Ns = case.stage_Ns()
        want = WANT_PLAN[case.plan]
        got = [regions_of(plan_chain(n, case.M, SXM_SMS, case.chain_q, case.taper), len(n)) for _, n in pieces_of(kinds, Ns)]
        assert got == want, (case.cid, got)


def test_want_plan_pins_match_plan_info():
    with_pins = 0
    for case in CASES:
        kinds, Ns = case.stage_Ns()
        with chain_options(case.chain, case.chain_q, case.taper):
            plans = [plan_info(n, case.M, k) for k, n in pieces_of(kinds, Ns)]
        if plans[0][0] != SXM_SMS:
            continue
        with_pins += 1
        assert [regions_of(p, len(n)) for p, (_, n) in zip(plans, pieces_of(kinds, Ns))] == WANT_PLAN[case.plan], case
    if with_pins == 0:
        pytest.skip('the plans are made for a device with other than 132 SMs')


def _cpu_policy(M, monkeypatch):
    """A policy whose parameters live on the host: only the host logic of the algorithms runs."""
    from promp_b200 import _lib
    from promp_b200.policies import MetaGaussianMLPPolicy
    monkeypatch.setattr(_lib, 'require_cuda', lambda: _lib.load())
    return MetaGaussianMLPPolicy(name='p', obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64), device='cpu')


def _cpu_algo(kind, M, S1, monkeypatch, explore=False):
    from promp_b200.meta_algos import ProMP, TRPOMAML
    pol = _cpu_policy(M, monkeypatch)
    if kind == 'promp':
        return pol, ProMP(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, learning_rate=1e-3,
                          num_ppo_steps=1, clip_eps=0.3, init_inner_kl_penalty=5e-4, adaptive_inner_kl_penalty=False)
    return pol, TRPOMAML(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, exploration=explore)


@pytest.mark.parametrize('algo_kind,S1,explore', [('promp', 3, False), ('promp', 4, False), ('trpo', 3, True),
                                                  ('trpo', 4, False), ('promp', 6, False)])
def test_long_chains_run_as_launches_of_at_most_six_stages(algo_kind, S1, explore, monkeypatch):
    """MAMLAlgo._meta_pass with three or more inner steps, host side only (every launch recorded, none run): the
    promp_policy_chain calls carry the whole stage list in order in pieces of at most six stages, and the launch re-use
    pointers of stage 0 go to the first piece only."""
    from promp_b200 import _lib
    from promp_b200.samplers.device_data import PhaseData
    M, N = 3, 200
    pol, algo = _cpu_algo(algo_kind, M, S1, monkeypatch, explore)
    calls = []

    def record(name, *args):
        if name in ('promp_policy_chain', 'promp_policy_chain_padded'):
            n, arr = args[5], args[6]
            st = (_lib.PolicyStage * n).from_address(arr.value)
            calls.append(dict(stages=[(s.kind, s.N, s.params, s.param_stride, s.grad, s.out_params, s.vec, s.out, s.obj_kind)
                                      for s in st], skip=(args[7], args[8]), ws=(args[9], args[10])))
        else:
            calls.append(dict(name=name))
    monkeypatch.setattr(_lib, 'call', record)
    monkeypatch.setattr(_lib, 'ptr', lambda t: None if t is None else t.data_ptr())
    monkeypatch.setattr(_lib, 'stream', lambda: None)
    phases = []
    for s in range(S1 + 1):
        ph = PhaseData(M, 1, N, 2, 2, torch.device('cpu'))
        ph.adv = torch.zeros(M, N)
        phases.append(ph)
    if explore:
        phases[-1].adj_avg_rewards_mean = torch.zeros(M)
    # the first pass after _adapt re-uses its launch: fake the cache _adapt_launch leaves
    P = pol.num_params
    algo._reuse_bufs = (torch.zeros(1, dtype=torch.int32), torch.zeros(P))
    algo._adapt_cache = dict(phase=phases[0], adv=phases[0].adv, gen=0, grad=torch.zeros(M, P), new=torch.zeros(M, P),
                             stats_all=algo._stats_rows(S1 + 1))
    if algo_kind == 'promp':
        algo._objective_pass(phases, want_grad=True, reduce=False)
    else:
        algo._meta_pass(pol.theta, phases, _lib.OBJ_RATIO, 0.0, [0.0] * S1, want_grad=True, reduce=explore,
                        explore=algo._explore(phases))
    assert algo._adapt_cache is None, 'the pass must have taken the re-use route'
    chains = [c for c in calls if 'stages' in c]
    kinds, _ = chain_kinds(S1, explore=explore)
    assert [len(c['stages']) for c in chains] == [min(MAX_STAGES, len(kinds) - i) for i in range(0, len(kinds), MAX_STAGES)]
    stages = [s for c in chains for s in c['stages']]
    assert [s[0] for s in stages] == kinds
    # order: each inner step starts from the previous one's out_params, the outer step from the last; each HVP takes the
    # previous direction vector and runs at the parameters of its inner step
    for s in range(1, S1 + 1):
        assert stages[s][2] == stages[s - 1][5], s
    for i, s in enumerate(range(S1 - 1, -1, -1)):
        h = stages[S1 + 1 + i]
        assert h[2] == stages[s][2] and h[3] == stages[s][3]
        assert h[6] == (stages[S1][4] if i == 0 else stages[S1 + i][7])
    if explore:
        assert stages[-1][8] == _lib.OBJ_EXPLORE and stages[-1][3] == 0
    assert chains[0]['skip'] == (algo._reuse_bufs[0].data_ptr(), algo._reuse_bufs[1].data_ptr())
    assert all(c['skip'] == (None, None) for c in chains[1:])
    assert len({c['ws'] for c in chains}) == 1, 'one workspace for every piece'
    # the workspace covers the largest piece
    lib = _lib.load()
    for k, n in pieces_of(kinds, [N] * len(kinds)):
        need = lib.promp_policy_chain_workspace_bytes(2, 2, 64, M, len(k), ctypes.cast(_stages(k, n), ctypes.c_void_p))
        assert 0 < need <= chains[0]['ws'][1]


@pytest.mark.parametrize('algo_kind', ['promp', 'trpo', 'vpg'])
def test_more_than_six_inner_steps_rejected_at_construction(algo_kind, monkeypatch):
    from promp_b200.meta_algos import ProMP, TRPOMAML, VPGMAML
    pol = _cpu_policy(2, monkeypatch)
    cls = dict(promp=ProMP, trpo=TRPOMAML, vpg=VPGMAML)[algo_kind]
    cls(policy=pol, inner_lr=0.1, meta_batch_size=2, num_inner_grad_steps=6)
    with pytest.raises(ValueError, match='num_inner_grad_steps=7: at most 6'):
        cls(policy=pol, inner_lr=0.1, meta_batch_size=2, num_inner_grad_steps=7)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _dist_info(case):
    if case.out_tanh:
        from test_output_tanh import otanh_dist_info_for
        return otanh_dist_info_for(case.act)
    if case.act == 'relu':
        from test_relu_policy import relu_dist_info
        return relu_dist_info
    return th.dist_info


class Setup(object):
    """The case's policy, algorithm, device phases and float64 host phases (per task: ragged phases differ in length)."""

    def __init__(self, case, nudge=True):
        from promp_b200.meta_algos import ProMP, TRPOMAML
        from promp_b200.policies import MetaGaussianMLPPolicy
        from promp_b200.samplers.device_data import PhaseData, RaggedPhaseData
        self.case = c = case
        M, Do, Da = c.M, c.Do, c.Da
        seed = 7000 + sum(map(ord, c.cid))
        rng = np.random.RandomState(seed)
        self.dims = (Do, Da, (64, 64))
        kw = dict(hidden_nonlinearity=c.act, output_nonlinearity='tanh' if c.out_tanh else None)
        self.pol = pol = MetaGaussianMLPPolicy(name='p', obs_dim=Do, action_dim=Da, meta_batch_size=M, hidden_sizes=(64, 64), **kw)
        theta = th.init_params(*self.dims, rng=rng).astype(np.float64) + 0.1 * rng.randn(th.num_params(*self.dims))
        theta[-Da:] = rng.uniform(-0.7, 0.0, size=Da)
        self.theta = theta.astype(np.float32)
        pol.set_params(self.theta)
        if c.algo == 'promp':
            self.algo = ProMP(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=c.S1, learning_rate=1e-3,
                              num_ppo_steps=1, clip_eps=po.CLIP_EPS, init_inner_kl_penalty=5e-3, adaptive_inner_kl_penalty=False)
        else:
            self.algo = TRPOMAML(policy=pol, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=c.S1, exploration=c.explore)
        self.algo.use_chain = True
        dist = _dist_info(c)
        t64 = torch.from_numpy(self.theta).double().view(1, -1).expand(M, -1)
        self.phases, self.cpus = [], []          # cpus[s][m]: dict of [1, n, .] float64 tensors
        for s in range(c.S1 + 1):
            nv = c.n_valid[s] if c.n_valid is not None else None
            N = c.phase_N(s)
            obs = rng.randn(M, N, Do)
            with torch.no_grad():
                mean, ls = dist(t64, torch.from_numpy(obs), self.dims, pol.min_log_std)
            old_mean = mean.numpy() + 0.1 * rng.randn(M, N, Da)
            old_ls = ls.numpy() + 0.05 * rng.randn(M, 1, Da)
            act = old_mean + np.exp(old_ls) * rng.randn(M, N, Da)
            adv = rng.randn(M, N)
            f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
            obs, act, adv, old_mean, old_ls = f(obs), f(act), f(adv), f(old_mean), f(old_ls)
            nvm = nv if nv is not None else [N] * M
            self.cpus.append([dict(obs=obs[m:m + 1, :n], act=act[m:m + 1, :n], adv=adv[m:m + 1, :n], mean=old_mean[m:m + 1, :n],
                                   log_std=np.broadcast_to(old_ls[m:m + 1], (1, n, Da)))
                              for m, n in enumerate(nvm)])
            if nv is not None:
                ph = RaggedPhaseData([[n] for n in nv], Do, Da, torch.device('cuda'))
                assert ph.N == N
                for m, n in enumerate(nv):             # poison in the padding rows, as the launcher tests do
                    obs[m, n:] = 1e3; act[m, n:] = -50.0; adv[m, n:] = 1e4; old_mean[m, n:] = 7.0
            else:
                ph = PhaseData(M, 1, N, Do, Da, torch.device('cuda'))
            ph.obs.copy_(torch.from_numpy(obs)); ph.act.copy_(torch.from_numpy(act)); ph.mean.copy_(torch.from_numpy(old_mean))
            ph.log_std.copy_(torch.from_numpy(old_ls[:, 0]))
            ph.adv = torch.from_numpy(adv).cuda()
            self.phases.append(ph)
        if c.explore:
            self.coeff = rng.randn(M).astype(np.float32)
            self.phases[-1].adj_avg_rewards_mean = torch.from_numpy(self.coeff).cuda()
        if nudge and c.act == 'relu':
            self._nudge_kinks(dist)
        if nudge and c.algo == 'promp':
            self._nudge_clip_ties(dist)

    def data(self, m):
        out = []
        for s, per in enumerate(self.cpus):
            d = {k: torch.from_numpy(np.ascontiguousarray(v)).double() for k, v in per[m].items()}
            if self.case.explore and s == self.case.S1:
                d['adj_avg_rewards'] = torch.full_like(d['adv'], float(self.coeff[m]))
            out.append(d)
        return out

    def _thetas(self, m):
        """float64 parameters [1, P] of task m at every inner step: theta_0 = theta, theta_{s+1} = the SGD step on phase s."""
        d = self.data(m)
        cur = torch.from_numpy(self.theta).double().view(1, -1).requires_grad_(True)
        out, clip0 = [cur.detach()], self.pol.min_log_std
        for s in range(self.case.S1):
            cur = th.adapt_sym(cur, d[s], self.dims, 0.1, min_log_std=clip0)[0].detach().requires_grad_(True)
            out.append(cur.detach())
            clip0 = None
        return out

    def _preacts(self, theta, obs):
        """Both hidden layers' pre-activations [1, n, 128] of the ReLU policy."""
        W0, b0, W1, b1 = th.split_params(theta, *self.dims)[:4]
        z1 = torch.matmul(obs, W0) + b0.unsqueeze(-2)
        return torch.cat([z1, torch.matmul(torch.relu(z1), W1) + b1.unsqueeze(-2)], -1)

    def _nudge_kinks(self, dist):
        """A ReLU pre-activation within float32 round-off of 0 can take the other side of the kink in float32 than in float64,
        and then its sample's whole contribution to the gradient differs.  Give every such sample a zero advantage, the way
        _nudge_clip_ties treats clip ties: phase s is judged at theta_s, the parameters every stage on phase s runs at.  The
        margin is 10x the largest |float32 - float64| pre-activation difference measured on the case's own data."""
        c = self.case
        adv_dev = [ph.adv.cpu().numpy() for ph in self.phases]
        for s in range(c.S1 + 1):
            z64, err = [], 0.0
            for m in range(c.M):
                t = self._thetas(m)[s]
                obs = torch.from_numpy(np.ascontiguousarray(self.cpus[s][m]['obs'])).double()
                z = self._preacts(t, obs)
                err = max(err, float((self._preacts(t.float(), obs.float()).double() - z).abs().max()))
                z64.append(z)
            eps = 10.0 * err
            for m in range(c.M):
                near = (z64[m].abs() < eps).any(-1).numpy()[0]
                self.cpus[s][m]['adv'] = self.cpus[s][m]['adv'].copy()
                self.cpus[s][m]['adv'][0, near] = 0.0
                adv_dev[s][m, :len(near)][near] = 0.0
        for ph, a in zip(self.phases, adv_dev):
            ph.adv.copy_(torch.from_numpy(a))

    def _nudge_clip_ties(self, dist):
        """An outer-phase sample whose float64 ratio lies within 1e-5 of 1 +- clip_eps could take the other branch of the
        clipped objective in float32: give it a zero advantage (on the device too)."""
        c = self.case
        adv_dev = self.phases[-1].adv.cpu().numpy()
        for m in range(c.M):
            d = self.data(m)
            cur = torch.from_numpy(self.theta).double().view(1, -1).requires_grad_(True)
            clip0 = self.pol.min_log_std
            for s in range(c.S1):
                cur = th.adapt_sym(cur, d[s], self.dims, 0.1, min_log_std=clip0)[0].detach().requires_grad_(True)
                clip0 = None
            with torch.no_grad():
                mean, ls = dist(cur, d[-1]['obs'], self.dims, clip0)
                r = th.likelihood_ratio(d[-1]['act'], d[-1]['mean'], d[-1]['log_std'], mean, ls).numpy()[0]
            tie = (np.abs(r - (1 - po.CLIP_EPS)) < 1e-5) | (np.abs(r - (1 + po.CLIP_EPS)) < 1e-5)
            self.cpus[-1][m]['adv'] = self.cpus[-1][m]['adv'].copy()
            self.cpus[-1][m]['adv'][0, tie] = 0.0
            adv_dev[m, :len(tie)][tie] = 0.0
        self.phases[-1].adv.copy_(torch.from_numpy(adv_dev))

    def oracle(self):
        """Per task: the float64 meta-gradient [M, P], outer surrogate [M], inner KLs [S1, M], outer KL [M]; with exploration
        the task-mean gradient [1, P] of the whole objective instead."""
        c, algo = self.case, self.algo
        kind = 'promp' if c.algo == 'promp' else 'trpo'
        coeff = list(algo.inner_kl_coeff) if c.algo == 'promp' else None
        grads, surr, ikl, okl = [], [], [], []
        for m in range(c.M):
            t64 = torch.tensor(self.theta, dtype=torch.float64, requires_grad=True)
            obj, kls, outer_kl = th.meta_objective(t64, self.data(m), self.dims, 0.1, kind, po.CLIP_EPS, coeff,
                                                   min_log_std=self.pol.min_log_std, exploration=c.explore)
            grads.append(torch.autograd.grad(obj, t64)[0].numpy())
            pen = float(torch.mean(torch.as_tensor(coeff, dtype=torch.float64) * kls)) if coeff and c.S1 else 0.0
            surr.append(float(obj.detach()) - pen)
            ikl.append(kls.detach().numpy())
            okl.append(float(outer_kl.detach()))
        g = np.stack(grads)
        if c.explore:
            g = g.mean(0, keepdims=True)
        return g, np.array(surr), np.stack(ikl, 1) if c.S1 else np.zeros((0, c.M)), np.array(okl)

    def run(self):
        """One evaluation: (gradient [M, P] per task, or [1, P] reduced with exploration; stats_all [S, M, 3])."""
        from promp_b200 import _lib
        c, algo, pol = self.case, self.algo, self.pol
        with chain_options(c.chain, c.chain_q, c.taper):
            if c.algo == 'promp':
                res = algo._objective_pass(self.phases, want_grad=True, reduce=False)
            else:
                res = algo._meta_pass(pol.theta, self.phases, _lib.OBJ_RATIO, 0.0, [0.0] * c.S1, want_grad=True,
                                      reduce=c.explore, explore=algo._explore(self.phases))
            torch.cuda.synchronize()
        g = res['grad'].view(1, -1) if c.explore else res['grad_tasks']
        return g.clone(), res['stats_all'][:, :, :3].clone()

    def ctrl_words(self):
        return self.algo._ws_chain[:ctrl_bytes(self.case.M) // 4].cpu().numpy()


def _check_plan(case, setup):
    """The device's plan is the case's pin (132 SMs) or the Python copy's plan at the device's SM count, and each piece runs
    as one dataflow launch."""
    from promp_b200 import _lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kinds, Ns = case.stage_Ns()
    pol = setup.pol
    with chain_options(case.chain, case.chain_q, case.taper):
        for i, (k, n) in enumerate(pieces_of(kinds, Ns)):
            got = plan_info(n, case.M, k)
            assert got[0] == sms
            assert got == plan_chain(n, case.M, sms, case.chain_q, case.taper, k)
            if sms == SXM_SMS:
                assert regions_of(got, len(n)) == WANT_PLAN[case.plan][i]
            st = _stages(k, n)
            launches = getattr(_lib.load(), pol.entries['chain_num_launches'])(case.Do, case.Da, pol.hidden_arg, case.M, len(k),
                                                                               ctypes.cast(st, ctypes.c_void_p))
            assert launches == (case.launches[i] if case.launches else 1), (case, i, launches)


def _check_against_oracle(setup, g, stats):
    c, pol = setup.case, setup.pol
    want, surr, ikl, okl = setup.oracle()
    mask = np.ones(pol.num_params, dtype=bool)
    mask[pol._pad_index_np] = False
    assert np.all(g.cpu().numpy()[:, mask] == 0.0), c.cid + ': pad entries of the gradient are not 0.0'
    po.assert_blocks(c.cid + ' meta-gradient', pol.unpad_flat(g.cpu().numpy()), want, c.Do, c.Da, 64)
    # stats: outer surrogate (not with exploration, whose term is not in that row), inner KLs, outer KL; the 1e-6 floor is
    # check_grad's 1e-6 x mean |term|, with unit-variance advantages and ratios near one
    st = stats.cpu().numpy().astype(np.float64)
    pairs = [(st[:c.S1, :, 1], ikl), (st[c.S1, :, 1], okl)]
    if not c.explore:
        pairs.append((st[c.S1, :, 0], surr))
    for got, w in pairs:
        assert np.all(np.abs(got - w) <= po.RTOL * np.abs(w) + 1e-6), (c.cid + ' stats', got, w)


_FIRST_PASS = {}


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c.cid for c in CASES])
def test_chain_case_against_float64(case, monkeypatch):
    po._cuda()
    monkeypatch.setattr(th, 'dist_info', _dist_info(case))
    setup = Setup(case)
    _check_plan(case, setup)
    if case.reuse:
        return _check_reuse(setup)
    g1, st1 = setup.run()
    g2, st2 = setup.run()
    assert torch.equal(g1, g2) and torch.equal(st1, st2), case.cid + ': not run-to-run bit-identical'
    assert (setup.ctrl_words() == 0).all(), case.cid + ': control words not left zero'
    _check_against_oracle(setup, g1, st1)


def _check_reuse(setup):
    """The first inner pass after _adapt skips stage 0 of the chain (skip_flag hit) and takes _adapt's outputs.  With
    _adapt's outputs replaced by the ones the chain computes for stage 0 itself, the re-use pass is bit-identical to the pass
    without re-use; with _adapt's own outputs it passes the float64 bar."""
    algo, pol = setup.algo, setup.pol
    recorded = []
    stage = algo._stage

    def recording_stage(kind, phase, params, stride, obj_kind, **kw):
        recorded.append(kw)
        return stage(kind, phase, params, stride, obj_kind, **kw)
    pol.switch_to_pre_update()
    algo.adapt_phase(setup.phases[0])
    assert algo._adapt_cache is not None
    g_reuse, st_reuse = setup.run()
    assert algo._adapt_cache is None, 'the pass did not take the re-use route'
    assert int(algo._reuse_bufs[0].item()) == 1, '_adapt must report an inactive step-0 clip'
    _check_against_oracle(setup, g_reuse, st_reuse)
    algo._stage = recording_stage
    try:
        g_plain, st_plain = setup.run()                  # no cache: stage 0 runs inside the chain
    finally:
        del algo._stage
    assert (setup.ctrl_words() == 0).all()
    g0, new0 = recorded[0]['grad'].clone(), recorded[0]['out_params'].clone()
    pol.switch_to_pre_update()
    algo.adapt_phase(setup.phases[0])
    cache = algo._adapt_cache
    cache['grad'].copy_(g0)
    cache['new'].copy_(new0)
    cache['stats_all'][0, :, :3].copy_(st_plain[0])
    g_hit, st_hit = setup.run()
    assert algo._adapt_cache is None and int(algo._reuse_bufs[0].item()) == 1
    assert torch.equal(g_hit, g_plain) and torch.equal(st_hit, st_plain), 're-use pass differs from the pass without re-use'
    assert (setup.ctrl_words() == 0).all()
    # a perturbed theta' in the cache must reach the output untouched: a kernel that recomputed stage 0 would overwrite it
    pol.switch_to_pre_update()
    algo.adapt_phase(setup.phases[0])
    cache = algo._adapt_cache
    bumped = new0 + 1e-2 * torch.sign(new0)
    cache['grad'].copy_(g0)
    cache['new'].copy_(bumped)
    g_bump, _ = setup.run()
    assert algo._adapt_cache is None and int(algo._reuse_bufs[0].item()) == 1
    assert torch.equal(cache['new'], bumped), 'stage 0 ran although the launch re-use flag was set'
    assert not torch.equal(g_bump, g_plain), 'the cached theta\' did not reach the output'


@pytest.mark.gpu
def test_chain_cases_in_reverse_order_on_one_workspace():
    """Every case once with its own workspace, then again in reverse order with one workspace shared by all of them (different
    M, stage counts and pieces): bit-identical outputs, control words zero after each."""
    po._cuda()
    cases = [c for c in CASES if not c.reuse]
    setups = [Setup(c, nudge=False) for c in cases]
    first = [s.run() for s in setups]
    ws = torch.zeros(max(s.algo._ws_chain.numel() for s in setups), dtype=torch.int32, device='cuda')
    for i in reversed(range(len(setups))):
        s = setups[i]
        s.algo._ws_chain = ws
        g, st = s.run()
        assert s.algo._ws_chain is ws
        assert torch.equal(g, first[i][0]) and torch.equal(st, first[i][1]), s.case.cid
        assert (ws[:ctrl_bytes(s.case.M) // 4].cpu().numpy() == 0).all(), s.case.cid


@pytest.mark.gpu
@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
def test_promp_three_inner_steps_trains_through_trainer(graph):
    """Seven-stage chains (two pieces) through the Trainer, eager and as a captured CUDA graph.  At M=4, N=200 (8 tiles) the
    automatic rule runs every piece as one launch per stage: the dataflow kernel's split chains are covered by
    test_chain_case_against_float64 (c10-*, c14-*)."""
    po._cuda()
    from promp_b200.envs import normalize, MetaPointEnvCorner
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler, MetaSampleProcessor
    from promp_b200.baselines import LinearFeatureBaseline
    from promp_b200.meta_algos import ProMP
    from promp_b200.meta_trainer import Trainer
    from promp_b200.utils import logger
    logger.set_quiet(True)
    np.random.seed(3)
    M, E, H, S1 = 4, 5, 40, 3
    env = normalize(MetaPointEnvCorner())
    policy = MetaGaussianMLPPolicy(name='p', obs_dim=2, action_dim=2, meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    proc = MetaSampleProcessor(baseline=LinearFeatureBaseline(), discount=0.99, gae_lambda=1, normalize_adv=True)
    algo = ProMP(policy=policy, inner_lr=0.1, meta_batch_size=M, num_inner_grad_steps=S1, learning_rate=1e-3, num_ppo_steps=2)
    th0 = policy.theta.clone()
    trainer = Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=proc, n_itr=2,
                      num_inner_grad_steps=S1, use_cuda_graph=graph)
    trainer.train()
    kv = logger.last_dump()
    assert np.isfinite(kv['LossAfter']) and np.isfinite(kv['Step_%d-AverageReturn' % S1])
    assert torch.isfinite(policy.theta).all() and not torch.equal(policy.theta, th0)
