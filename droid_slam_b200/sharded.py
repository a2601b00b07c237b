"""Edge-sharded dense BA across GPUs (one process per GPU, torch.distributed for the plumbing).

The factor graph is partitioned by SOURCE frame: rank r owns a contiguous range of frames and every edge whose
source frame `ii` lies in it (SURVEY.md section 8e).  Everything per edge (corr lookup, Jacobian blocks) and the depth
elimination of an owned frame (C_k, w_k, E_k are sums over the out-edges of k) is then rank-local.  The only exchange
per Gauss-Newton iteration is ONE all-reduce (sum) of the reduced pose system [6P x 6P | 6P] in fp64; the damped
Cholesky solve is replicated (bit-identical inputs -> identical dx on every rank, no broadcast), the depth update is
local to the owner, and the owners' inverse depths are exchanged once after the last iteration.

The reference has no counterpart (its only collective is DDP training, train.py:28-36).
"""
import ctypes

import torch
import torch.distributed as dist

from . import c_api

__all__ = ["partition_frames", "shard_edges", "CApiEngine", "ShardedBA", "P2PSystem"]


def partition_frames(ii, n_frames, world):
    """contiguous frame ranges [lo,hi) per rank, balanced by out-degree (= per-rank edge count). Deterministic."""
    deg = torch.bincount(ii.cpu(), minlength=n_frames).double()
    total = float(deg.sum())
    csum = torch.cumsum(deg, 0)
    bounds = [0]
    for r in range(1, world):
        target = total * r / world
        cut = int(torch.searchsorted(csum, torch.tensor(target, dtype=csum.dtype)).item()) + 1
        cut = max(cut, bounds[-1])
        bounds.append(min(cut, n_frames))
    bounds.append(n_frames)
    return [(bounds[r], bounds[r + 1]) for r in range(world)]


def shard_edges(ii, lo, hi):
    """indices of the edges owned by the rank holding frames [lo,hi) (original order kept)."""
    return torch.nonzero((ii >= lo) & (ii < hi)).reshape(-1)


class P2PSystem:
    """peer-visible buffers for the fused reduction of the pose system (DESIGN.md section 6): every rank allocates two slots of
    36P^2+6P doubles plus 8 flags in symmetric memory (torch.distributed._symmetric_memory) and learns its peers' mapped pointers"""

    def __init__(self, n, device, group=None):
        import torch.distributed._symmetric_memory as symm_mem
        self.nd = n * n + n
        self.buf = symm_mem.empty(2 * self.nd + 8, dtype=torch.float64, device=device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        torch.cuda.synchronize(device)
        dist.barrier(group)
        self.ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.world = int(self.hdl.world_size)
        self.rank = int(self.hdl.rank)
        self.epoch = 0
        # the epoch VALUE lives on the device (advanced by the signal kernel), which makes a whole step CUDA-graph capturable; the
        # host counter only alternates the two slots, so a captured graph must contain an even number of GN iterations
        self.epoch_dev = torch.zeros(1, dtype=torch.int64, device=device)
        assert self.world <= 8


class CApiEngine:
    """the three phases of the C ABI (include/droid_b200.h) on one GPU"""

    def __init__(self, device):
        self.L = c_api.load()
        self.device = torch.device(device)
        self.args = None

    def setup(self, poses, disps, intrinsics, disps_sens, targets, weights, eta_by_frame, ii, jj, t0, t1, lm, ep, own, p2p=None):
        N, ht, wd = disps.shape
        E = ii.shape[0]
        L = self.L
        self.ws_bytes = L.dba_ba_workspace_bytes(N, E, ht, wd, t0, t1)
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=self.device)
        self.P = t1 - t0
        n = 6 * self.P
        off = L.dba_ba_system_offset(N, E, ht, wd, t0, t1)
        self.system = self.ws[off:off + 8 * (n * n + n)].view(torch.float64)      # the all-reduce buffer, in place
        self.dx = torch.zeros(self.P, 6, device=self.device)
        self.dz = torch.zeros(N, ht * wd, device=self.device)                      # at most one depth frame per frame
        a = c_api.ba_args(poses, disps, intrinsics, disps_sens, targets, weights, eta_by_frame, ii, jj, t0, t1, lm, ep, self.dx, self.dz,
                          self.ws, torch.cuda.current_stream(self.device).cuda_stream, own=own, eta_by_frame=True)
        self.p2p = p2p
        if p2p is not None:
            assert p2p.nd == n * n + n, "P2PSystem was sized for another window"
            a.p2p_world, a.p2p_rank = p2p.world, p2p.rank
            for k, ptr in enumerate(p2p.ptrs):
                a.p2p_system[k] = ptr
            a.p2p_epoch_dev = p2p.epoch_dev.data_ptr()
        self.args = a
        self._keep = (poses, disps, intrinsics, disps_sens, targets, weights, eta_by_frame, ii, jj)
        c_api.check(L.dba_ba_prepare(ctypes.byref(a)), "ba_prepare")

    def build(self):
        if self.p2p is not None:          # next epoch on every rank: selects the slot and is what the peers wait for
            self.p2p.epoch += 1
            self.args.p2p_epoch = self.p2p.epoch
        c_api.check(self.L.dba_ba_build(ctypes.byref(self.args)), "ba_build")
        return self.system

    def publish(self):
        """fused path: release-store this rank's epoch into every peer's flag array (after build, before solve)"""
        c_api.check(self.L.dba_ba_p2p_signal(ctypes.byref(self.args)), "ba_p2p_signal")

    def solve(self):
        c_api.check(self.L.dba_ba_solve(ctypes.byref(self.args)), "ba_solve")


class ShardedBA:
    """host-side driver of an edge-sharded BA; `engine` provides setup/build/solve for the local shard"""

    def __init__(self, engine, group=None, p2p=None):
        self.engine = engine
        self.group = group
        self.p2p = p2p          # P2PSystem: fuse the all-reduce into the Cholesky kernel's load phase over NVLink peer memory
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.allreduce_bytes = 0

    def run(self, poses, disps, intrinsics, disps_sens, targets, weights, eta_by_frame, ii, jj, t0, t1, iterations, lm, ep, bounds,
            exchange_disps=True):
        """poses/disps are the full (replicated) state; targets/weights/ii/jj are this rank's edge shard.
        In place on poses (all ranks identical) and disps (owned frames; all frames after the final exchange)."""
        own = bounds[self.rank]
        if self.p2p is not None:
            self.engine.setup(poses, disps, intrinsics, disps_sens, targets, weights, eta_by_frame, ii, jj, t0, t1, lm, ep, own, p2p=self.p2p)
        else:
            self.engine.setup(poses, disps, intrinsics, disps_sens, targets, weights, eta_by_frame, ii, jj, t0, t1, lm, ep, own)
        self.allreduce_bytes = 0
        for _ in range(iterations):
            system = self.engine.build()
            if self.p2p is not None:
                self.engine.publish()                 # no collective call: the solve kernel sums the peers' copies itself
            elif self.world > 1:
                dist.all_reduce(system, op=dist.ReduceOp.SUM, group=self.group)     # the one exchange per GN iteration
                self.allreduce_bytes += system.numel() * system.element_size()
            self.engine.solve()
        if exchange_disps and self.world > 1:
            # owners' inverse depths: during the iterations a rank only reads and writes the rows it owns, so the other rows can be
            # zeroed and ONE all-reduce (sum) rebuilds the full tensor in place on every rank
            lo, hi = own
            if lo > 0:
                disps[:lo].zero_()
            if hi < disps.shape[0]:
                disps[hi:].zero_()
            dist.all_reduce(disps, op=dist.ReduceOp.SUM, group=self.group)
        return poses, disps
