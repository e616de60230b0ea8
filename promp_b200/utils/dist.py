"""torch.distributed plumbing: the path shards by task, the only data-path collective is the sum
all-reduce of the flat meta-gradient [P] (plus a packed vector of logged scalars)."""


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist
    return None


_p2p = None       # P2PComm once enable_p2p_allreduce() has run


def allreduce_sum_(t):
    """Sum over ranks, in place.  float32 CUDA vectors that fit the P2P buffer go through promp_allreduce_p2p (one
    kernel over NVLink peer memory, rank-ordered, CUDA-graph capturable); everything else through NCCL."""
    d = _dist()
    if d is None:
        return t
    if _p2p is not None and _p2p.accepts(t):
        return _p2p.allreduce_(t)
    d.all_reduce(t, op=d.ReduceOp.SUM)
    return t


class P2PComm(object):
    """Peer-memory all-reduce plumbing: one IPC-exported buffer per rank (csrc/comm.cu)."""

    def __init__(self, capacity_floats):
        import ctypes
        import torch
        from promp_b200 import _lib
        d = _dist()
        assert d is not None, "P2PComm needs an initialised multi-rank process group"
        self.rank, self.world, self.cap = d.get_rank(), d.get_world_size(), int(capacity_floats)
        self.device = torch.device('cuda', torch.cuda.current_device())
        lib = _lib.load()
        nbytes = lib.promp_comm_buffer_bytes(self.world, self.cap)
        own = ctypes.c_void_p()
        _lib.check(lib.promp_comm_alloc(nbytes, ctypes.byref(own)), 'promp_comm_alloc')
        handle = ctypes.create_string_buffer(64)
        _lib.check(lib.promp_ipc_get_handle(own, handle), 'promp_ipc_get_handle')
        blobs = [None] * self.world
        d.all_gather_object(blobs, bytes(handle.raw))
        ptrs = []
        for r, blob in enumerate(blobs):
            if r == self.rank:
                ptrs.append(own.value)
            else:
                peer = ctypes.c_void_p()
                _lib.check(lib.promp_ipc_open_handle(ctypes.create_string_buffer(blob, 64), ctypes.byref(peer)),
                           'promp_ipc_open_handle')
                ptrs.append(peer.value)
        self._own, self._ptrs = own, ptrs
        self.peers = torch.tensor(ptrs, dtype=torch.int64, device=self.device)
        self.epoch = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.ticket = torch.zeros(1, dtype=torch.int32, device=self.device)     # completion ticket of the multi-CTA all-reduce
        d.barrier()

    def accepts(self, t):
        import torch
        return t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and 0 < t.numel() <= self.cap

    def allreduce_(self, t, scale=1.0):
        from promp_b200 import _lib
        _lib.call('promp_allreduce_p2p', self.world, self.rank, t.numel(), self.cap, _lib.ptr(t), _lib.ptr(t), float(scale),
                  _lib.ptr(self.peers), _lib.ptr(self.epoch), _lib.ptr(self.error), _lib.ptr(self.ticket), _lib.stream())
        return t

    def check(self):
        if int(self.error.item()) != 0:
            raise RuntimeError("promp_allreduce_p2p: a peer rank did not arrive within the time-out")


def enable_p2p_allreduce(capacity_floats=8192):
    """Route small float32 all-reduces through the NVLink peer-memory kernel (needed for CUDA-graph replay at N > 1)."""
    global _p2p
    if _dist() is not None and _p2p is None:
        _p2p = P2PComm(capacity_floats)
    return _p2p


def world_size():
    d = _dist()
    return d.get_world_size() if d is not None else 1


def rank():
    d = _dist()
    return d.get_rank() if d is not None else 0


def shard_tasks(all_tasks, rank, world):
    """Rank `rank` of `world` owns the contiguous slice of the global task list (every rank draws the same
    list from the same numpy seed, so every rank gets the tasks a one-GPU run gives it).  With the fused samplers
    the samples do not depend on the number of GPUs either (MetaSampler: global Philox keys and reset draws, the
    early-termination cut over all ranks); the step loop over host-reset envs keeps per-rank reset draws, and the
    meta-gradient all-reduce sums in a rank-dependent order (last-bit differences)."""
    n = len(all_tasks)
    assert n % world == 0, "global meta batch must be divisible by the number of ranks"
    per = n // world
    return list(all_tasks[rank * per:(rank + 1) * per])
