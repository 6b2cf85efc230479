"""P virtual ranks of the sharded PageRank and WCC on one GPU (test harness).

PageRank: every virtual rank is a CudaShardBackend of the same graph with its own x[2], score vector and
error share, all on the current stream.  A sweep runs the ranks' steps one after another and then
exchanges the finished out_scores in one of two ways:
  * host copies: each rank's rows are copied into every other rank's x_next (what the NCCL all-gather
    does between GPUs; the kernels run PEERS = false);
  * peer stores: every rank's step gets the other ranks' x_next as peer pointers and k_pr_sell /
    k_pr_finish store each finished out_score into them (PEERS = true; on one device a peer pointer is
    a plain pointer, and the ranks never run at the same time).
Shared by test_gpu_parity.py, test_gpu_pr_paths.py and test_gpu_shard_paths.py."""
from __future__ import annotations

import numpy as np
import torch

from graph_b200 import _capi
from graph_b200.multigpu import CudaShardBackend, CudaWccBackend, owner_of_rows, vertex_ranges


class VirtualRanks:
    def __init__(self, g, world: int, damping: float = 0.85):
        self.g, self.world, self.damping = g, world, damping
        self.n = n = g.node_count()
        self.ranks = [CudaShardBackend(g, r, world) for r in range(world)]
        self.n_active = self.ranks[0].n_active
        dev = self.ranks[0].device
        owner = torch.from_numpy(owner_of_rows(np.arange(n), world)).to(dev)
        self.mine = [owner == r for r in range(world)]
        self.x = [[torch.zeros(n, dtype=torch.float32, device=dev) for _ in range(2)] for _ in range(world)]
        self.scores = [torch.empty(n, dtype=torch.float32, device=dev) for _ in range(world)]
        self.err = [torch.zeros(1, dtype=torch.float64, device=dev) for _ in range(world)]
        self.sweep = 0

    def init(self):
        for r, b in enumerate(self.ranks):
            b.init(self.damping, self.x[r][0], self.x[r][1], self.scores[r])
        self.sweep = 0

    def step(self, peers: bool = False):
        """One sweep on every rank, in rank order, then the exchange; returns the ranks' error shares."""
        self.sweep += 1
        cur, nxt = (self.sweep - 1) & 1, self.sweep & 1
        for r, b in enumerate(self.ranks):
            ptrs = [self.x[q][nxt].data_ptr() for q in range(self.world) if q != r] if peers else None
            b.step(self.damping, self.sweep, self.x[r][cur], self.x[r][nxt], ptrs, self.scores[r], self.err[r])
        torch.cuda.current_stream().synchronize()
        if not peers:
            for r in range(self.world):  # the all-gather: every rank's rows go to every other rank
                for q in range(self.world):
                    if q != r:
                        self.x[q][nxt][self.mine[r]] = self.x[r][nxt][self.mine[r]]
        return [float(e.item()) for e in self.err]

    def x_next(self):
        return [x[self.sweep & 1] for x in self.x]

    def run(self, sweeps: int, tolerance: float = 0.0, peers: bool = False):
        """init + sweeps until the rank-order sum of the shares is below `tolerance` (when > 0) or `sweeps`
        have run; returns the total error of the last sweep"""
        self.init()
        while True:
            total = 0.0
            for e in self.step(peers):
                total += e
            if (tolerance > 0.0 and total < tolerance) or self.sweep == sweeps:
                return total

    def scores_host(self):
        """every rank's score vector holds its own rows (rows without in-edges: rank 0) and zeros elsewhere"""
        full = torch.stack(self.scores).sum(dim=0)
        return self.ranks[0].finish(full).cpu().numpy()


def wcc_virtual_ranks(g, world: int, **cfg):
    """The phases of ShardedWcc.run on `world` virtual ranks: every rank runs them on its vertex range over
    its own full parent array, and the all-gather is a list of snapshots.  Returns (parents, labels)."""
    b = CudaWccBackend(g, **cfg)
    ranges = vertex_ranges(g.node_count(), world)
    parents = [b.new_parent() for _ in range(world)]

    def merge_all():
        snap = [p.clone() for p in parents]
        for r, p in enumerate(parents):
            for q in range(world):
                if q != r:
                    b.phase(_capi.WCC_MERGE, p, other=snap[q])
            b.phase(_capi.WCC_COMPRESS, p)

    for r, p in enumerate(parents):
        b.phase(_capi.WCC_INIT, p)
        b.phase(_capi.WCC_SAMPLE, p, *ranges[r])
        b.phase(_capi.WCC_COMPRESS, p)
    merge_all()
    labels = [b.sample_label(p) for p in parents]
    for r, p in enumerate(parents):
        b.phase(_capi.WCC_LINK_REMAINING, p, *ranges[r], labels[r][0], labels[r][1])
        b.phase(_capi.WCC_COMPRESS, p)
    merge_all()
    return parents, labels
