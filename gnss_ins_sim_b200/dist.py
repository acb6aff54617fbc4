"""Multi-GPU plumbing: Monte-Carlo runs shard embarrassingly across ranks (one process
per GPU, torch.distributed); the only data-path collectives are one broadcast of the
CPU-generated trajectory and the exchange of the final error statistics
(SURVEY 8e).  Works un-initialised (single process) and with the gloo backend (CPU
tests of the host logic); on GPUs the backend is NCCL over NVLink.

Statistics are combined from each rank's (count, max|e|, mean, std) by Chan's pairwise update
(merge_stats), as robust as np.std's two passes: inside K3x through NVLink peer memory
(P2PStats), or after ONE all_gather (StatsMerger, combine_local_stats).
"""
import numpy as np
import torch
import torch.distributed as td


def initialised():
    return td.is_available() and td.is_initialized()


def rank():
    return td.get_rank() if initialised() else 0


def world():
    return td.get_world_size() if initialised() else 1


def shard(total, r=None, w=None):
    """Contiguous block [lo, hi) of `total` runs owned by rank r of w (first ranks take the
    remainder).  Global run ids are rank-independent, so results do not depend on w."""
    if r is None and w is None and not initialised():
        return 0, int(total)
    r = rank() if r is None else r
    w = world() if w is None else w
    base, rem = divmod(int(total), w)
    lo = r * base + min(r, rem)
    return lo, lo + base + (1 if r < rem else 0)


def _comm_device():
    if initialised() and td.get_backend() == 'nccl':
        return torch.device('cuda', torch.cuda.current_device())
    return torch.device('cpu')


def all_reduce(t, op):
    """all-reduce a tensor in place on the backend's device; returns it on its own device."""
    if not initialised():
        return t
    dev = _comm_device()
    buf = t if t.device == dev else t.to(dev)
    td.all_reduce(buf, op=op)
    if buf is not t:
        t.copy_(buf)
    return t


def merge_stats(blocks):
    """Chan et al. pairwise merge of per-rank (count, max|e|, mean, std) -> (max, mean, std) of
    the union, as robust as np.std's two passes.  blocks: iterable of (n, max[nc], mean[nc],
    std[nc]) numpy; empty shards (n = 0) are skipped.  Non-finite shard statistics merge as
    NumPy's statistics of the union are: np.maximum keeps a NaN max, a NaN std stays NaN,
    and a +-inf mean stays +-inf (NaN against the other sign or a NaN)."""
    n_a, mx_a, mean_a, m2_a = 0, None, None, None
    for n_b, mx_b, mean_b, std_b in blocks:
        n_b = int(n_b)
        if n_b == 0:
            continue
        m2_b = np.asarray(std_b, dtype=np.float64) ** 2 * n_b
        if n_a == 0:
            n_a, mx_a, mean_a, m2_a = n_b, np.array(mx_b, dtype=np.float64), \
                np.array(mean_b, dtype=np.float64), m2_b
            continue
        n = n_a + n_b
        with np.errstate(invalid='ignore'):
            delta = mean_b - mean_a
            # a +-inf or NaN mean on either side: the sum of the means, +-inf or NaN as
            # np.mean of the union is
            mean_a = np.where(np.isfinite(delta), mean_a + delta * (n_b / n),
                              mean_a + mean_b)
            m2_a = m2_a + m2_b + delta * delta * (n_a * n_b / n)
        mx_a = np.maximum(mx_a, mx_b)
        n_a = n
    return np.stack([mx_a, mean_a, np.sqrt(m2_a / n_a)]), n_a


_mergers = {}
_p2p = {}


def fused_exchange(ncomp=9):
    """A cached P2PStats for the WORLD group, or None if symmetric memory is unavailable (every
    rank must call this the same number of times: construction is collective)."""
    key = (ncomp, world())
    if key not in _p2p:
        obj = None
        if initialised() and td.get_backend() == 'nccl':
            try:
                obj = P2PStats(ncomp)
            except Exception:
                obj = None
            # all ranks or none: a rank on which the set-up failed must not leave the others spinning
            ok = torch.tensor([1 if obj is not None else 0], dtype=torch.int32, device=_comm_device())
            td.all_reduce(ok, op=td.ReduceOp.MIN)
            if int(ok.item()) == 0:
                obj = None
        _p2p[key] = obj
    return _p2p[key]


def combine_local_stats(stats, local_runs):
    """stats [3, nc] = (max|e|, mean, std) of this rank's `local_runs` runs (numpy; anything if
    local_runs == 0) -> [3, nc] of all ranks' runs: ONE all_gather of 3 nc + 1 doubles."""
    stats = np.ascontiguousarray(stats, dtype=np.float64)
    if not initialised():
        return stats
    key = (stats.shape[1], world(), str(_comm_device()))
    if key not in _mergers:
        _mergers[key] = StatsMerger(stats.shape[1])
    m = _mergers[key]
    return m(torch.from_numpy(stats).to(m.dev), local_runs)


class StatsMerger:
    """combine_local_stats with everything preallocated and the shard statistics left on the
    device until after the collective: one tiny pack, ONE all_gather, one D2H, Chan merge."""

    def __init__(self, ncomp=9):
        self.nc = ncomp
        self.dev = _comm_device()
        self.mine = torch.zeros(3 * ncomp + 1, dtype=torch.float64, device=self.dev)
        self.outs = torch.zeros((world(), 3 * ncomp + 1), dtype=torch.float64, device=self.dev)

    def __call__(self, stats_dev, local_runs):
        """stats_dev: CUDA/CPU tensor [3, nc] on the collective's device (or None)."""
        nc = self.nc
        if not initialised():
            return stats_dev.cpu().numpy()
        if local_runs:
            self.mine[:3 * nc].copy_(stats_dev.reshape(-1), non_blocking=True)
        self.mine[3 * nc] = float(local_runs)
        if td.get_backend() == 'nccl':
            td.all_gather_into_tensor(self.outs.view(-1), self.mine)
        else:   # gloo (CPU tests of the host logic)
            td.all_gather(list(self.outs.unbind(0)), self.mine)
        host = self.outs.cpu().numpy()
        blocks = [(row[3 * nc], row[0:nc], row[nc:2 * nc], row[2 * nc:3 * nc]) for row in host]
        return merge_stats(blocks)[0]


class P2PStats:
    """K3x: shard statistics + exchange + merge in ONE kernel per rank over NVLink peer memory
    (b2ins_error_stats_exchange_f64).  torch's symmetric memory supplies the peer-mapped
    windows (plumbing); the kernel, the flags and the merge are ours.  Raises if symmetric
    memory cannot be set up (callers fall back to StatsMerger / NCCL)."""

    def __init__(self, ncomp=9):
        import ctypes
        import torch.distributed._symmetric_memory as symm
        from . import _lib
        assert initialised() and td.get_backend() == 'nccl'
        self._lib, self._check = _lib.load(), _lib.check
        self.nc, self.w, self.r = ncomp, world(), rank()
        dev = torch.device('cuda', torch.cuda.current_device())
        group = td.group.WORLD
        try:
            symm.enable_symm_mem_for_group(group.group_name)
        except Exception:
            pass
        self.win = symm.empty((2 * self.w * 32,), dtype=torch.float64, device=dev)
        self.win.zero_()
        self.hdl = symm.rendezvous(self.win, group)
        ptrs = [int(x) for x in self.hdl.buffer_ptrs]
        assert len(ptrs) == self.w
        self.ptrs = (ctypes.c_uint64 * self.w)(*ptrs)
        self.out = torch.zeros((3, ncomp), dtype=torch.float64, device=dev)
        self.flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self.empty = torch.zeros((1, ncomp), dtype=torch.float64, device=dev)
        self.seq = 0
        torch.cuda.synchronize()
        td.barrier()                      # every window is zeroed before anyone's first store

    def __call__(self, end_err, local_runs, stream_ptr=None):
        """end_err: CUDA f64 [local_runs, nc] tensor or a raw device address (ignored if
        local_runs == 0); stream_ptr: raw cudaStream_t (default: torch's current stream)
        -> CUDA [3, nc]."""
        import ctypes
        self.seq += 1
        if not local_runs:
            ptr = self.empty.data_ptr()
        else:
            ptr = end_err.data_ptr() if isinstance(end_err, torch.Tensor) else int(end_err)
        stream = ctypes.c_void_p(stream_ptr if stream_ptr is not None
                                 else torch.cuda.current_stream().cuda_stream)
        self._check(self._lib.b2ins_error_stats_exchange_f64(
            int(local_runs), self.nc, ctypes.c_void_p(ptr), self.r, self.w, self.ptrs,
            self.seq, ctypes.c_void_p(self.out.data_ptr()), ctypes.c_void_p(self.flag.data_ptr()),
            stream))
        return self.out

    def timed_out(self):
        return bool(self.flag.item())

    def reset_timeout(self):
        self.flag.zero_()


def gather_rows(local, total_runs):
    """Concatenate per-rank row blocks [R_local, C] (shard() order) -> numpy [total, C] on
    every rank.  Blocks are padded to the largest shard for the all_gather."""
    if not initialised():
        return local.cpu().numpy()
    w = world()
    sizes = [shard(total_runs, r, w) for r in range(w)]
    cap = max(hi - lo for lo, hi in sizes)
    cols = torch.tensor([0 if local is None else local.shape[1]], dtype=torch.int64,
                        device=_comm_device())
    all_reduce(cols, td.ReduceOp.MAX)
    C = int(cols.item())
    dev = _comm_device()
    pad = torch.zeros((cap, C), dtype=torch.float64, device=dev)
    if local is not None and local.shape[0]:
        pad[:local.shape[0]] = local.to(dev)
    outs = [torch.empty_like(pad) for _ in range(w)]
    td.all_gather(outs, pad)
    return np.concatenate([o[:hi - lo].cpu().numpy() for o, (lo, hi) in zip(outs, sizes)], axis=0)


def broadcast_trajectory(traj, src=0):
    """Rank `src` holds the CPU-generated trajectory dict of (n,3) arrays; everyone gets it."""
    if not initialised():
        return traj
    names = ['ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro']
    dev = _comm_device()
    n = torch.tensor([traj['ref_gyro'].shape[0] if rank() == src else 0], dtype=torch.int64,
                     device=dev)
    td.broadcast(n, src)
    buf = torch.empty((int(n.item()), 15), dtype=torch.float64, device=dev)
    if rank() == src:
        buf.copy_(torch.from_numpy(np.concatenate([traj[k] for k in names], axis=1)))
    td.broadcast(buf, src)
    host = buf.cpu().numpy()
    out = {k: np.ascontiguousarray(host[:, 3 * i:3 * i + 3]) for i, k in enumerate(names)}
    if traj is not None:
        for k in ('time', 'ini'):
            if k in traj:
                out[k] = traj[k]
    return out
