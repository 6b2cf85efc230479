"""Multi-GPU PageRank: 1-D edge-cut across the GPUs of one box, one process per GPU.

The reference has no distributed code at all (SURVEY.md §2.3); this is the one exchange step
BASELINE.json's north_star adds.  The JACOBI path orders rows by in-degree; its 32-row slices are
dealt round-robin over the ranks (rank p owns slices p, p+P, ...), so every rank holds the same mix
of hub and tail rows and builds the layout of its own rows only (`gb_pr_shard_create`).  Every rank
sweeps its rows (`gb_pr_shard_step`) and the finished out_scores are exchanged either

  * "peer"      — fused: the sweep kernels store each finished out_score straight into every rank's
                  next vector — one `multimem.st` replicated by the NVSwitch when torch symmetric
                  memory offers a multicast mapping, else one NVLink store per peer; the inter-sweep
                  barrier and the sum of the ranks' error shares are one tiny kernel over peer-mapped
                  control blocks (`gb_pr_shard_sync`): no collective and no host round trip per sweep, or
  * "allgather" — baseline: the own slices are packed and exchanged with one NCCL all-gather.

`torch.distributed` is plumbing only; the compute is the same CUDA kernels as on one GPU.  The
compute backend is injectable so that the orchestration (deal, exchange, stop rule, assembly) is
testable with gloo on CPUs (tests/test_multigpu_gloo.py).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import _capi
from ._capi import check, lib

SLICE = 32  # rows per dealt slice (one SELL slice / one warp of the finish kernel)


def owner_of_rows(rows, world: int):
    """Rank owning each internal row under the cyclic deal of 32-row slices."""
    return (np.asarray(rows, dtype=np.int64) // SLICE) % world


class CudaShardBackend:
    """The product backend: gb_pr_shard_* of libgraph_b200.so on this rank's GPU."""

    def __init__(self, graph, rank: int, world: int):
        self.graph = graph
        self.rank, self.world = rank, world
        self.n = graph.node_count()
        self.device = torch.device("cuda", torch.cuda.current_device())
        self._shard = C.c_void_p()
        self.launches = 0
        check(lib.gb_pr_shard_create(graph._g, rank, world, C.byref(self._shard)))
        self.stats = self.info()
        self.n_active = self.stats["active_rows"]

    @classmethod
    def from_handle(cls, handle, rank: int, world: int, n: int, device):
        """A backend around a shard built elsewhere (gb_pr_shards_csr_u32), which it now owns and frees; the
        shard holds no graph."""
        self = cls.__new__(cls)
        self.graph = None
        self.rank, self.world, self.n = rank, world, n
        self.device = torch.device(device)
        self._shard = handle if isinstance(handle, C.c_void_p) else C.c_void_p(handle)
        self.launches = 0
        self.stats = self.info()
        self.n_active = self.stats["active_rows"]
        return self

    def info(self) -> dict:
        st = _capi.PrShardStats()
        check(lib.gb_pr_shard_info(self._shard, C.byref(st)))
        return st.as_dict()

    def plan_shape(self) -> dict:
        """Diagnostics: the launch shape of this shard's sweep kernels."""
        sh = _capi.PrPlanShape()
        check(lib.gb_pr_shard_plan_shape(self._shard, C.byref(sh)))
        return sh.as_dict()

    def __del__(self):
        sh, self._shard = getattr(self, "_shard", None), None
        if sh:
            try:
                lib.gb_pr_shard_free(sh)
            except Exception:
                pass

    @staticmethod
    def _stream() -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def init(self, damping, x0, x1, scores):
        check(lib.gb_pr_shard_init(self._shard, damping, C.c_void_p(x0.data_ptr()), C.c_void_p(x1.data_ptr()),
                                   C.c_void_p(scores.data_ptr()), self._stream()))
        self.launches += 1

    def step(self, damping, sweep_no, x_cur, x_next, peer_ptrs, scores, err, mc_ptr=0):
        arr = None
        if peer_ptrs:
            arr = (C.c_void_p * len(peer_ptrs))(*peer_ptrs)
        check(lib.gb_pr_shard_step(self._shard, damping, sweep_no, C.c_void_p(x_cur.data_ptr()),
                                   C.c_void_p(x_next.data_ptr()), arr, len(peer_ptrs or ()),
                                   C.c_void_p(mc_ptr) if mc_ptr else None,
                                   C.c_void_p(scores.data_ptr()), C.c_void_p(err.data_ptr()), self._stream()))
        self.launches += self.stats["launches_per_sweep"] + (1 if sweep_no == 1 else 0)

    def sync(self, seq, err_local, self_block, peer_blocks, total_err, slot):
        """Device-side barrier + error sum (gb_pr_shard_sync); peer_blocks has one entry per rank."""
        arr = (C.c_void_p * len(peer_blocks))(*peer_blocks)
        check(lib.gb_pr_shard_sync(self._shard, seq, C.c_void_p(err_local.data_ptr()), C.c_void_p(self_block), arr,
                                   C.c_void_p(total_err.data_ptr()), slot, self._stream()))
        self.launches += 1

    def finish(self, scores_internal):
        out = torch.empty_like(scores_internal)
        check(lib.gb_pr_shard_finish(self._shard, C.c_void_p(scores_internal.data_ptr()), C.c_void_p(out.data_ptr()),
                                     self._stream()))
        self.launches += 1
        return out


class ShardedPageRank:
    """page_rank over `world` shards; every rank ends up with the full score vector.

    run(max_iterations, damping, tolerance) follows page_rank.rs:88-110: sweep, error = sum over all
    ranks, stop when error < tolerance or the sweep count reaches max_iterations.
    """

    def __init__(self, graph=None, exchange: str = "auto", backend=None, group=None, multicast: bool = True):
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.backend = backend if backend is not None else CudaShardBackend(graph, self.rank, self.world)
        b = self.backend
        self.n, self.n_active = b.n, b.n_active
        # vectors are padded so that the dealt slices form a full (slices, world, 32) grid
        grid = SLICE * self.world
        self.n_pad = (self.n + grid - 1) // grid * grid
        self.active_pad = min(self.n_pad, (self.n_active + grid - 1) // grid * grid)
        dev = b.device
        self.exchange = "allgather" if exchange in ("nccl", "allgather") else exchange
        self._peer_next = [None, None]
        self._mc_next = [0, 0]
        self.multicast = False
        self.diag = None
        self.x = None
        if exchange in ("auto", "peer") and dev.type == "cuda" and self.world > 1:
            try:
                self._setup_symmetric(dev, multicast)
                self.exchange = "peer"
            except Exception as exc:  # symmetric memory unavailable: fall back to the NCCL exchange
                if exchange == "peer":
                    raise
                self._symm_error = repr(exc)
        if self.exchange == "auto":
            self.exchange = "allgather"
        if self.x is None:
            self.x = [torch.zeros(self.n_pad, dtype=torch.float32, device=dev) for _ in range(2)]
        self.scores = torch.zeros(self.n, dtype=torch.float32, device=dev)
        self.err = torch.zeros(1, dtype=torch.float64, device=dev)
        self.ran_iterations = 0
        self.error = 0.0

    # -- symmetric memory (NVLink peer mappings, NVSwitch multicast) --
    def _setup_symmetric(self, dev, multicast):
        import torch.distributed._symmetric_memory as symm_mem
        group_name = (self.group or dist.group.WORLD).group_name
        ctl_floats = 64  # this rank's 192-byte control block of the device-side barrier (gb_pr_shard_sync)
        buf = symm_mem.empty(2 * self.n_pad + ctl_floats, dtype=torch.float32, device=dev)
        hdl = symm_mem.rendezvous(buf, group_name)
        self._symm = (buf, hdl)
        buf.zero_()
        torch.cuda.synchronize()
        dist.barrier(group=self.group)   # every control block is zero before anybody publishes into it
        self.x = [buf[: self.n_pad], buf[self.n_pad: 2 * self.n_pad]]
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        self._sync_blocks = [p + 2 * self.n_pad * 4 for p in ptrs]
        self._sync_seq = 0
        self._total_err = torch.zeros(64, dtype=torch.float64, device=dev)
        mc = int(getattr(hdl, "multicast_ptr", 0) or 0) if multicast else 0
        self.multicast = mc != 0
        for which in (0, 1):
            off = which * self.n_pad * 4
            self._peer_next[which] = [ptrs[p] + off for p in range(self.world) if p != self.rank]
            self._mc_next[which] = mc + off if mc else 0

    @property
    def launches(self) -> int:
        return getattr(self.backend, "launches", 0)

    def rebind(self, graph):
        """Point the same exchange state (symmetric buffers, control blocks) at a new graph of the same
        node count: the old shard layout is released, the new graph's shard is built (collective: every
        rank rebinds).  Used by the end-to-end path, where nothing of a graph stays resident."""
        if graph.node_count() != self.n:
            raise ValueError("rebind needs a graph with the same node count")
        launches = self.launches
        self.backend = None            # frees the old shard before the new layout is allocated
        self.backend = CudaShardBackend(graph, self.rank, self.world)
        self.backend.launches = launches
        if self.backend.n_active != self.n_active:
            self.n_active = self.backend.n_active
            grid = SLICE * self.world
            self.active_pad = min(self.n_pad, (self.n_active + grid - 1) // grid * grid)
        return self

    def _exchange(self, x_next):
        if self.exchange == "peer":
            return  # the kernels already stored this rank's values into every peer
        # own slices (rank, rank + world, ...) packed, one all-gather, unpacked in place
        k = self.active_pad // (SLICE * self.world)
        if k == 0:
            return
        grid = x_next[: self.active_pad].view(k, self.world, SLICE)
        mine = grid[:, self.rank, :].contiguous()
        out = torch.empty((self.world * k, SLICE), dtype=x_next.dtype, device=x_next.device)
        dist.all_gather_into_tensor(out, mine, group=self.group)
        grid.copy_(out.view(self.world, k, SLICE).permute(1, 0, 2))

    def run(self, max_iterations: int = 20, damping: float = 0.85, tolerance: float = 0.0):
        b = self.backend
        b.init(damping, self.x[0][: self.n], self.x[1][: self.n], self.scores)
        # fused exchange: no barrier is needed before sweep 1 — a peer's init and this rank's sweep-1
        # stores touch disjoint entries (init writes x0, scores and the rows without in-edges of x1), and
        # every later hazard is ordered by the device barrier that ends each sweep
        device_sync = self.exchange == "peer" and hasattr(b, "sync")
        sweep = 0
        limit = max_iterations if max_iterations else 100000
        diag = self.diag
        while True:
            sweep += 1
            cur, nxt = self.x[(sweep - 1) & 1], self.x[sweep & 1]
            peers = self._peer_next[sweep & 1] if self.exchange == "peer" else None
            mc = self._mc_next[sweep & 1] if self.exchange == "peer" else 0
            if diag is not None:
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                ev[0].record()
            if mc:
                b.step(damping, sweep, cur, nxt, peers, self.scores, self.err, mc)
            else:
                b.step(damping, sweep, cur, nxt, peers, self.scores, self.err)
            if diag is not None:
                ev[1].record()
            self._exchange(nxt)
            if diag is not None:
                ev[2].record()
                diag.append(ev)
            # total error of the sweep; also the barrier that orders the peer stores of sweep k before
            # any rank's reads in sweep k+1
            if device_sync:
                slot = sweep % 64
                b.sync(self._sync_seq + sweep, self.err, self._sync_blocks[self.rank], self._sync_blocks,
                       self._total_err, slot)
                total = self._total_err[slot]
            else:
                dist.all_reduce(self.err, op=dist.ReduceOp.SUM, group=self.group)
                total = self.err[0]
            if tolerance > 0.0:
                self.error = float(total.item())
                if self.error < tolerance:
                    break
            if sweep == limit:
                break
        self.ran_iterations = sweep
        if device_sync:
            self._sync_seq += sweep
        if not tolerance > 0.0:
            self.error = float(total.item())
        return self

    def diag_summary(self):
        """(mean kernel ms, mean exchange ms) per sweep of the recorded run (diagnostics only)."""
        torch.cuda.synchronize()
        k = [a.elapsed_time(b) for a, b, _ in self.diag]
        x = [b.elapsed_time(c) for _, b, c in self.diag]
        return float(np.mean(k)), float(np.mean(x))

    def scores_device(self):
        """Full score vector in original ids on this rank's device: every rank's score vector holds its
        own rows and zeros elsewhere, so one sum all-reduce assembles the full vector."""
        full = self.scores.clone()
        if self.world > 1:
            dist.all_reduce(full, op=dist.ReduceOp.SUM, group=self.group)
        return self.backend.finish(full)

    def scores_host(self, reuse: bool = False) -> np.ndarray:
        """Full score vector on the host.  reuse=True copies into one page-locked buffer owned by this
        object (overwritten by the next call) instead of a fresh pageable array: the end-to-end path reads
        268 MB per step at RMAT-26."""
        full = self.scores_device()
        if not (reuse and full.is_cuda):
            return full.cpu().numpy()
        host = getattr(self, "_host_scores", None)
        if host is None or host.numel() != full.numel():
            try:
                host = torch.empty(full.numel(), dtype=full.dtype, pin_memory=True)
            except RuntimeError:
                host = torch.empty(full.numel(), dtype=full.dtype)
            self._host_scores = host
        host.copy_(full, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return host.numpy()


# =====================================================================================================
# Multi-GPU WCC (1-D cut by vertex range)
# =====================================================================================================
def vertex_ranges(n: int, world: int):
    """Contiguous, 32-aligned vertex ranges of (almost) equal size; Graph500 ids are scrambled, so equal
    ranges carry (almost) equal numbers of edges."""
    cuts = [min(n, ((n * p // world) + 31) // 32 * 32) for p in range(world)] + [n]
    return [(cuts[p], max(cuts[p], cuts[p + 1])) for p in range(world)]


class CudaWccBackend:
    """gb_wcc_shard_phase / gb_wcc_sample_label of libgraph_b200.so on this rank's GPU."""

    def __init__(self, graph, neighbor_rounds=2, sampling_size=1024, chunk_size=16384):
        self.graph = graph
        self.n = graph.node_count()
        self.cfg = _capi.WccConfig(chunk_size, neighbor_rounds, sampling_size)
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.launches = 0

    def new_parent(self):
        return torch.empty(self.n, dtype=torch.int32, device=self.device)

    def phase(self, which, parent, vb=0, ve=0, skip=0, use_skip=0, other=None):
        check(lib.gb_wcc_shard_phase(self.graph._g, C.byref(self.cfg), which, vb, ve, skip, int(use_skip),
                                     C.c_void_p(parent.data_ptr()),
                                     C.c_void_p(other.data_ptr()) if other is not None else None,
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        self.launches += 1

    def sample_label(self, parent):
        label, found = C.c_uint32(0), C.c_int(0)
        check(lib.gb_wcc_sample_label(self.graph._g, C.byref(self.cfg), C.c_void_p(parent.data_ptr()),
                                      C.byref(label), C.byref(found),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return int(label.value), bool(found.value)


class ShardedWcc:
    """wcc_afforest over `world` ranks: every rank runs the phases of wcc() (wcc.rs:158-183) on its
    vertex range over a full parent[n]; the P forests are exchanged with one all-gather after the
    sampling phase and one after link_remaining, and merged with the Afforest link rule, so every rank
    ends with the same labels = minimum node id per component (bit-equal to the single-GPU result).

    The giant component that link_remaining skips is chosen on the MERGED sampled forest: skipping a
    vertex is only sound when both endpoints of each skipped edge are already connected or the other
    endpoint is processed by its owner, which a rank-local choice cannot guarantee."""

    def __init__(self, graph=None, backend=None, group=None, **cfg):
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.backend = backend if backend is not None else CudaWccBackend(graph, **cfg)
        self.n = self.backend.n
        self.vb, self.ve = vertex_ranges(self.n, self.world)[self.rank]
        self.timing = {}

    def _merge_all(self, parent):
        """All-gather the P forests and link every other rank's tree edges into ours."""
        b = self.backend
        if self.world == 1:
            return
        gathered = torch.empty((self.world, self.n), dtype=parent.dtype, device=parent.device)
        dist.all_gather_into_tensor(gathered.view(-1), parent, group=self.group)
        for q in range(self.world):
            if q != self.rank:
                b.phase(_capi.WCC_MERGE, parent, other=gathered[q])
        b.phase(_capi.WCC_COMPRESS, parent)

    def run(self):
        b = self.backend
        parent = b.new_parent()
        b.phase(_capi.WCC_INIT, parent)
        b.phase(_capi.WCC_SAMPLE, parent, self.vb, self.ve)
        b.phase(_capi.WCC_COMPRESS, parent)
        self._merge_all(parent)
        label, found = b.sample_label(parent)   # same forest, same seed: the same label on every rank
        b.phase(_capi.WCC_LINK_REMAINING, parent, self.vb, self.ve, label, found)
        b.phase(_capi.WCC_COMPRESS, parent)
        self._merge_all(parent)
        return parent
