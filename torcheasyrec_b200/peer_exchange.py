"""Host side of csrc/tzk_peer.cu: the sharded sparse step over peer memory (exchange="peer" in shard_model).

`enable_peer_exchange(sharded_collection, batch_size)` re-routes a `ShardedEmbeddingBagCollection` /
`ShardedEmbeddingCollection` from the NCCL all-to-alls to peer-memory kernels over the NVSwitch domain.  Per dim
group and per step (DESIGN.md §6):

    forward    ONE kernel on the compute stream: the requester gathers rows straight out of the owners' arenas
               (symmetric memory) and pools in bag order — bit-identical to the unsharded gather, any bag length.
    prep       (training; side stream, overlaps the rest of the forward pass)  tzk_peer_bucketize: stable multi-split of
               the local ids by destination into this rank's own wire buffers -> barrier A -> the owner pulls its chunk
               of every source's keys straight into the radix sort's input and sorts (tzk_fused_bwd_sort_peer).
    backward   publish the gradient (symmetric buffer; MEAN bags pre-divided) -> barrier B -> side stream: the run /
               update kernels fetch every gradient slice from the SOURCE rank's buffer in place
               (tzk_fused_bwd_apply_peer, 1/W gradient scale, App. A.6) -> barrier C (tables quiescent, wire buffers and
               gradient reusable); the stream is joined when the backward pass ends.
    dense      `PeerDenseGradSync`: publish the flat dense gradient -> barrier D -> every rank sums all W buffers in rank
               order (same bits everywhere) — no NCCL call anywhere in the step.

Symmetric allocations and the address exchange come from `torch.distributed._symmetric_memory` (plumbing, with a CUDA
IPC fallback); every kernel on the path is ours.  The whole step stays capturable: every barrier's epoch lives on the
device.  Wire capacity: `cap = static_capacity * max over destinations of the expected ids per step` (table-wise
features send everything to one owner, row-wise ones 1/W to each); an overflow drops ids, raises the device flag
`g.overflow` on EVERY rank in the same step (the owners read the sources' flags) and `check_overflow()` reports it.
"""
import ctypes
import os
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import functional as Fn
from .kernels import POOL_MEAN, build_layout
from .sparse import JaggedTensor, KeyedTensor


class _Symm:
    """One symmetric allocation: `t` is this rank's tensor, `ptrs` a host array with every rank's address as mapped in
    this process (rank order).  Allocation + address exchange: `torch.distributed._symmetric_memory` (cuMem VMM handles);
    TZK_PEER_ALLOC=ipc — or a failing rendezvous — falls back to classic CUDA IPC handles through
    torch.multiprocessing's reductions (cudaIpcGetMemHandle / cudaIpcOpenMemHandle), one all_gather_object each."""

    def __init__(self, numel: int, dtype, device, group) -> None:
        W = dist.get_world_size(group)
        n = max(int(numel), 1)
        self.h = None
        if os.environ.get("TZK_PEER_ALLOC", "symm") != "ipc":
            try:
                import torch.distributed._symmetric_memory as symm_mem

                self.t = symm_mem.empty(n, dtype=dtype, device=device)
                self.t.zero_()
                self.h = symm_mem.rendezvous(self.t, group)
                self.ptrs = (ctypes.c_uint64 * W)(*[int(p) for p in self.h.buffer_ptrs])
                return
            except Exception as e:  # noqa: BLE001 — e.g. no pidfd / fabric handle support in this container
                import warnings

                warnings.warn(f"symmetric-memory rendezvous failed ({e!r}); falling back to CUDA IPC handles")
        self._ipc(n, dtype, device, group, W)

    def _ipc(self, n: int, dtype, device, group, W: int) -> None:
        from torch.multiprocessing.reductions import reduce_tensor

        me = dist.get_rank(group)
        self.t = torch.zeros(n, dtype=dtype, device=device)
        torch.cuda.synchronize()
        fn, args = reduce_tensor(self.t)
        gathered = [None] * W
        dist.all_gather_object(gathered, args, group=group)
        self.peers = [self.t if r == me else fn(*gathered[r]) for r in range(W)]
        for r, pt in enumerate(self.peers):     # first touch enables peer access between the two devices
            if r != me:
                _ = pt[:1].to(device)
        torch.cuda.synchronize()
        self.ptrs = (ctypes.c_uint64 * W)(*[int(pt.data_ptr()) for pt in self.peers])


class _Site:
    """One barrier site: its own flag array (symmetric) and device epoch, so that sites on different streams never
    share a counter."""

    def __init__(self, owner: "PeerBase") -> None:
        self.pads = owner._alloc(owner.W, torch.int32)
        self.epoch = torch.zeros(1, dtype=torch.int32, device=owner.device)


class PeerBase:
    """Process / device plumbing shared by the sparse states and the dense gradient sync.  tests/
    test_peer_exchange_model.py swaps `_alloc`, `_host_barrier`, `_barrier` and the stream hooks for an in-process
    model (ranks = threads)."""

    def __init__(self, group, device, world: Optional[int] = None, rank: Optional[int] = None) -> None:
        self.group = group
        self.device = torch.device(device)
        self.W = int(world) if world is not None else dist.get_world_size(group)
        self.me = int(rank) if rank is not None else dist.get_rank(group)

    def _alloc(self, numel: int, dtype) -> "_Symm":
        return _Symm(numel, dtype, self.device, self.group)

    def _host_barrier(self) -> None:
        torch.cuda.synchronize()
        dist.barrier(group=self.group)

    def _barrier(self, site: _Site) -> None:
        Fn.backend().peer_barrier(site.pads, self.me, self.W, site.epoch)

    # ---- streams (no-ops off CUDA) ---------------------------------------------------------------------------------
    def _side_stream(self):
        if self.device.type != "cuda":
            return None
        st = getattr(self, "_side", None)
        if st is None:
            st = self._side = torch.cuda.Stream(device=self.device)
        return st

    def _on_side(self, fn) -> None:
        """Runs fn() on the side stream, ordered after everything enqueued on the current stream so far."""
        side = self._side_stream()
        if side is None:
            fn()
            return
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fn()

    def _join_side(self) -> None:
        side = self._side_stream()
        if side is not None:
            torch.cuda.current_stream().wait_stream(side)


def expected_load(g, plan, ids_per_feature: Sequence[int]) -> int:
    """max over destinations of the ids a step sends there (table-wise: everything to the owner; row-wise: 1/W each)."""
    from .distributed import TABLE_WISE

    W = g.world
    load = [0.0] * W
    for f, t in enumerate(g.local._feat_table):
        sh = plan[g.configs[t].name]
        if sh.kind == TABLE_WISE:
            load[sh.owner] += ids_per_feature[f]
        else:
            blocks = min(W, -(-g.configs[t].num_embeddings // sh.block))    # ranks that hold rows of this table
            for r in range(blocks):
                load[r] += ids_per_feature[f] / blocks
    return int(max(load)) + 1


class PeerState(PeerBase):
    """Peer-memory state of one `_DimGroup` (all tables of one embedding dim) of a pooled or sequence collection."""

    def __init__(self, g, plan, group, batch_size: int, ids_per_feature: Optional[Sequence[int]] = None) -> None:
        super().__init__(group, g.device, g.world, g.rank)
        self.g, self.B, self.pooled = g, int(batch_size), bool(g.pooled)
        dev, F, W = g.device, g.F, g.world
        lay = g.local.layout
        alpha = float(g.static_alpha or 1.5)
        # every rank's arena layout (deterministic from the plan: no communication)
        from .distributed import local_rows

        per_rank = [build_layout([local_rows(c, plan[c.name], r) for c in g.configs], g.local._table_dim,
                                 g.local._feat_table, list(lay.pool)) for r in range(W)]
        assert per_rank[self.me].w_off == list(lay.w_off), "local layout differs from the plan's"
        self.rf_w_off = torch.tensor([o for lr in per_rank for o in lr.w_off], dtype=torch.int64, device=dev)
        self.rf_key_base = torch.tensor([k for lr in per_rank for k in lr.key_base], dtype=torch.int64, device=dev)
        self.feat_rows = torch.tensor([g.configs[t].num_embeddings for t in g.local._feat_table], dtype=torch.int64,
                                      device=dev)
        # the arena moves into symmetric memory (same size on every rank: the largest shard), in the collection's table
        # dtype (FP16 tables: halfs; everything else of the exchange stays fp32)
        self.tables = self._alloc(max(lr.arena_elems for lr in per_rank), g.local.weights.dtype)
        n = g.local.weights.numel()
        self.tables.t[:n].copy_(g.local.weights.data)
        g.local.weights.data = self.tables.t[:n]
        self.bwd_mode = os.environ.get("TZK_PEER_BWD", "push")
        self._init_mirror(plan, per_rank)
        # id budget per step: one id per bag unless the caller knows better (sequence features: B * sequence_length)
        per_f = list(ids_per_feature) if ids_per_feature is not None else [self.B] * F
        self.max_nnz = int(sum(per_f))
        self.idx_span = F * self.B if self.pooled else max(self.max_nnz, 1)
        self._init_small_bwd(plan, per_rank)
        wire_f = [0 if (self.small is not None and self.small["is_small"][f]) else n for f, n in enumerate(per_f)]
        self.cap = (int(alpha * expected_load(g, plan, wire_f)) + 8) // 8 * 8
        self.cap = min(self.cap, (int(sum(wire_f)) + 8) // 8 * 8)     # a destination never gets more than everything
        assert W * self.idx_span < 2 ** 31 and W * self.cap < 2 ** 31
        g.static_nnz, g.static_cap = self.max_nnz, self.cap
        self.wire_key = self._alloc(W * self.cap, torch.int64)
        self.wire_idx = self._alloc(W * self.cap, torch.int32)
        self.counts = self._alloc(W + 1, torch.int32)
        # backward transport: "push" (default) = every source writes its gradient slices into the owners' receive
        # buffers in wire order (coalesced NVLink writes, the update then runs on local memory); "pull" = the sources
        # publish their gradient and the owners' update kernels read the 64-B slices over NVLink in place
        if self.bwd_mode == "push":
            self.recv = self._alloc(W * self.cap * g.dim, torch.float32)
            self._dummy_off = torch.zeros(2, dtype=torch.int64, device=dev)
        else:
            self.grad = self._alloc(self.B * g.total_dim if self.pooled else self.max_nnz * g.dim, torch.float32)
        self.site_a, self.site_b, self.site_c, self.site_b2 = _Site(self), _Site(self), _Site(self), _Site(self)
        self._ws = None
        self._prep_pending = False
        self._host_barrier()                 # flags are zero and tables are in place everywhere before the first step

    # ---- small tables: a per-step local copy ---------------------------------------------------------------------
    def _init_mirror(self, plan, per_rank) -> None:
        """Tables of at most TZK_PEER_MIRROR_ROWS rows (default 65536; 0 switches it off) are copied whole from their
        owners at the start of every forward pass — a few MB of long sequential NVLink reads — and looked up locally;
        only the big tables' rows cross NVLink as random 64-B reads.  Exact: the copy is taken after the barrier that
        closes the previous step's updates."""
        from .distributed import local_rows

        g, dev = self.g, self.device
        thr = int(os.environ.get("TZK_PEER_MIRROR_ROWS", "65536"))
        self.mirror = None
        self.feat_mirror_off = None
        self._m_off = {}
        if thr <= 0 or self.W == 1:
            return
        m_off, o = {}, 0
        for t, c in enumerate(g.configs):
            if c.num_embeddings <= thr:
                m_off[t] = o
                o += c.num_embeddings * c.embedding_dim
        if not m_off:
            return
        seg_rank, seg_src, seg_dst, seg_n = [], [], [], []
        first_feat = {}
        for f, t in enumerate(g.local._feat_table):
            first_feat.setdefault(t, f)
        for t, base in m_off.items():
            c = g.configs[t]
            sh = plan[c.name]
            for r in range(self.W):
                n = local_rows(c, sh, r)
                if n:
                    start = 0 if sh.kind == "table_wise" else r * sh.block
                    seg_rank.append(r)
                    seg_src.append(per_rank[r].w_off[first_feat[t]])
                    seg_dst.append(base + start * c.embedding_dim)
                    seg_n.append(n * c.embedding_dim)
        self._m_off = m_off
        self.mirror = torch.zeros(max(o, 4), dtype=g.local.weights.dtype, device=dev)     # (FP16 tables: halfs)
        self.feat_mirror_off = torch.tensor([m_off.get(t, -1) for t in g.local._feat_table], dtype=torch.int64, device=dev)
        self._seg = (torch.tensor(seg_rank, dtype=torch.int32, device=dev), torch.tensor(seg_src, dtype=torch.int64, device=dev),
                     torch.tensor(seg_dst, dtype=torch.int64, device=dev), torch.tensor(seg_n, dtype=torch.int64, device=dev))

    def _init_small_bwd(self, plan, per_rank) -> None:
        """Backward of the mirrored (small) tables: every rank reduces its OWN batch's gradients per row into a dense
        symmetric buffer (the fused backward's sort + run kernels with TZK_OPT_ACCUM_OUT), the owners add the W
        partial sums in rank order and update (tzk_peer_small_update).  69 % of Criteo's gradient rows never cross
        NVLink; what crosses is a few MB of sequential reads.  TZK_PEER_SMALL_BWD=0 sends every row over the wire."""
        import numpy as np

        from .distributed import local_rows
        from .kernels import FeatureLayout

        g, dev = self.g, self.device
        self.small = None
        self.feat_block_wire = g.feat_block
        lay = g.local.layout
        if (self.mirror is None or self.bwd_mode != "push" or os.environ.get("TZK_PEER_SMALL_BWD", "1") == "0"
                or any(d % 4 or d > 128 for d in lay.dim) or not lay.vec_ok):
            return
        m_off = self._m_off
        kb, k = {}, 0
        for t in sorted(m_off, key=lambda t: m_off[t]):
            kb[t] = k
            k += g.configs[t].num_embeddings
        ft = g.local._feat_table
        is_small = [t in m_off for t in ft]
        sl = FeatureLayout(
            w_off=[m_off.get(t, 0) for t in ft], rows=[g.configs[t].num_embeddings if t in m_off else 0 for t in ft],
            dim=list(lay.dim), col=list(lay.col), pool=list(lay.pool), key_base=[kb.get(t, -1) for t in ft],
            total_keys=max(k, 1), total_dim=lay.total_dim, arena_elems=self.mirror.numel()).to(dev)
        rec = np.dtype([("kb", "<i8"), ("start", "<i8"), ("w_off", "<i8"), ("psum_off", "<i8"), ("key_base", "<i8"),
                        ("first", "<i4"), ("n", "<i4"), ("dim", "<i4"), ("pad", "<i4")])
        first_feat = {}
        for f, t in enumerate(ft):
            first_feat.setdefault(t, f)
        rows, first = [], 0
        for t in sorted(m_off, key=lambda t: m_off[t]):
            c = g.configs[t]
            sh = plan[c.name]
            n = local_rows(c, sh, self.me)
            if n:
                start = 0 if sh.kind == "table_wise" else self.me * sh.block
                f = first_feat[t]
                rows.append((kb[t], start, lay.w_off[f], m_off[t], lay.key_base[f], first, n, c.embedding_dim, 0))
                first += n
        tabs = np.array(rows, dtype=rec) if rows else np.zeros(0, dtype=rec)
        blk = g.feat_block.clone()
        blk[torch.tensor(is_small, device=dev)] = 0
        self.feat_block_wire = blk
        self.small = dict(
            is_small=is_small, layout=sl, n_tabs=len(rows), total_rows=first,
            tabs=torch.from_numpy(tabs.view(np.uint8).copy()).to(dev) if rows else torch.zeros(8, dtype=torch.uint8, device=dev),
            psum=self._alloc(self.mirror.numel(), torch.float32), flags=self._alloc(max(k, 1), torch.int32), ws=None)

    def _small_ws(self, nnz: int, weighted: bool = False) -> torch.Tensor:
        k = Fn.backend()
        n = max(nnz, self.max_nnz)
        # (weighted bags: the id half also leaves the bag of every id and the sorted weights in the workspace)
        need = (k.fused_bwd_workspace_bytes(self.small["layout"], n, weighted=True) if weighted
                else k.fused_bwd_workspace_bytes(self.small["layout"], n))
        ws = self.small["ws"]
        if ws is None or ws.numel() < need:
            ws = self.small["ws"] = torch.empty(max(need, 256), dtype=torch.uint8, device=self.device)
        return ws

    # ---- weighted bags ---------------------------------------------------------------------------------------------
    def _weights(self, psw: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        """The per-sample weights this step uses: None for un-pooled collections (they ignore weights, like the nobag
        TBE).  They never leave this rank: its gather pools w * row and its push sends w * g (/ L); the owners' update
        is the unweighted one.  Host-side checks only (no device sync)."""
        if psw is None or not self.pooled:
            return None
        if psw.requires_grad:
            raise NotImplementedError("sharded EmbeddingBagCollection: per-sample weights that require grad (feature "
                                      "processors) are not supported; the weights of a weighted id feature are data")
        if self.bwd_mode != "push":
            raise NotImplementedError("weighted id features on a sharded EmbeddingBagCollection need the push transport "
                                      "of the peer exchange (TZK_PEER_BWD=push, the default): with pull the owners "
                                      "would need every source's weights")
        return psw

    # ---- forward ---------------------------------------------------------------------------------------------------
    def gather(self, ids: torch.Tensor, offsets: torch.Tensor, psw: Optional[torch.Tensor] = None,
               B: Optional[int] = None) -> torch.Tensor:
        """psw: the local batch's per-sample weights (weighted bags) or None.  B: the local batch when it is smaller
        than the one the exchange was sized for — only forward-only steps do that (the gather reads peer tables and
        needs no other rank's counts; the wire buffers of the backward are sized for self.B)."""
        g, k = self.g, Fn.backend()
        B = self.B if B is None else int(B)
        if B > self.B:
            raise RuntimeError(f"peer exchange is sized for local batches of {self.B} samples, got {B}")
        if ids.numel() > self.max_nnz:
            raise RuntimeError(f"peer exchange is sized for {self.max_nnz} ids per step, got {ids.numel()}")
        psw = self._weights(psw)
        wkw = {} if psw is None else {"per_sample_weights": psw}
        sel = self._split_lists() if self.pooled else None
        if sel is not None:
            # two launches over complementary feature lists: the one whose rows cross NVLink starts first, on its own
            # stream; the mirror refresh and the mirrored features' lookup run next to it
            out = torch.empty((B, g.local.layout.total_dim), dtype=torch.float32, device=ids.device)
            gs = self._gather_stream()
            cur = torch.cuda.current_stream() if gs is not None else None

            def remote():
                k.peer_pooled_gather_fwd(self.tables, self.rf_w_off, self.feat_rows, g.feat_block, g.feat_owner,
                                         g.local.layout, ids, offsets, B, self.W, out, self.mirror,
                                         self.feat_mirror_off, feat_sel=sel[1], **wkw)

            if gs is not None:
                gs.wait_stream(cur)
                with torch.cuda.stream(gs):
                    remote()
            else:
                remote()
            k.peer_mirror_refresh(self.tables, self.W, *self._seg, self.mirror)
            k.peer_pooled_gather_fwd(self.tables, self.rf_w_off, self.feat_rows, g.feat_block, g.feat_owner,
                                     g.local.layout, ids, offsets, B, self.W, out, self.mirror, self.feat_mirror_off,
                                     feat_sel=sel[0], **wkw)
            if gs is not None:
                cur.wait_stream(gs)
            return out
        if self.mirror is not None:
            k.peer_mirror_refresh(self.tables, self.W, *self._seg, self.mirror)
        if self.pooled:
            return k.peer_pooled_gather_fwd(self.tables, self.rf_w_off, self.feat_rows, g.feat_block, g.feat_owner,
                                            g.local.layout, ids, offsets, B, self.W, None, self.mirror,
                                            self.feat_mirror_off, **wkw)
        return k.peer_seq_gather_fwd(self.tables, self.rf_w_off, self.feat_rows, g.feat_block, g.feat_owner,
                                     g.local.layout, ids, offsets, B, self.W, self.mirror, self.feat_mirror_off)

    def _split_lists(self):
        """(mirrored features, features whose rows live in the owners' arenas) as device int32 lists, or None when the
        lookup stays one launch (no mirror, one of the lists empty, or TZK_PEER_SPLIT_GATHER off — the split has not been
        through a GPU validation pass yet: on with TZK_PEER_SPLIT_GATHER=1 / TZK_EXPERIMENTAL=1)."""
        sl = getattr(self, "_split_sel", False)
        if sl is False:
            from .kernels import _unvalidated_switch

            sl = None
            if self.mirror is not None and _unvalidated_switch("TZK_PEER_SPLIT_GATHER"):
                ft = self.g.local._feat_table
                loc = [f for f, t in enumerate(ft) if t in self._m_off]
                rem = [f for f, t in enumerate(ft) if t not in self._m_off]
                if loc and rem:
                    sl = (torch.tensor(loc, dtype=torch.int32, device=self.device),
                          torch.tensor(rem, dtype=torch.int32, device=self.device))
            self._split_sel = sl
        return sl

    def _gather_stream(self):
        if self.device.type != "cuda":
            return None
        st = getattr(self, "_gstream", None)
        if st is None:
            st = self._gstream = torch.cuda.Stream(device=self.device)
        return st

    def _workspace(self) -> torch.Tensor:
        k = Fn.backend()
        need = k.fused_bwd_workspace_bytes(self.g.local.layout, self.W * self.cap)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(max(need, 256), dtype=torch.uint8, device=self.device)
        return self._ws

    def prep(self, ids: torch.Tensor, offsets: torch.Tensor, psw: Optional[torch.Tensor] = None) -> None:
        """Id half of the backward (side stream): bucketize -> barrier A -> pull + sort at the owner.  psw (weighted
        bags): the bucketize also records every wire slot's weight in `wire_w` for this rank's push, and the small
        tables' sort keeps the weights in sorted order."""
        g, k = self.g, Fn.backend()
        psw = self._weights(psw)
        wkw = {}
        if psw is not None:
            if getattr(self, "wire_w", None) is None:    # local memory (only this rank's push reads it): no collective
                self.wire_w = torch.zeros(max(self.W * self.cap, 1), dtype=torch.float32, device=self.device)
            wkw = {"per_sample_weights": psw, "wire_w": self.wire_w}

        def run():
            if self._prep_pending:            # a forward pass without a backward: peers may still be pulling
                self._barrier(self.site_c)
            k.peer_bucketize(ids, offsets, g.F, self.B, self.W, self.feat_block_wire, g.feat_owner, self.feat_rows,
                             self.rf_key_base, self.pooled, self.cap, self.wire_key.t, self.wire_idx.t, self.counts.t,
                             **wkw)
            if self.small is not None:        # small tables: this rank's own ids, sorted by (table, row)
                self.small["flags"].t.zero_()
                if psw is not None:
                    k.fused_bwd_sort(self.pooled, self.small["layout"], ids, offsets, self.B,
                                     self._small_ws(ids.numel(), weighted=True), per_sample_weights=psw)
                else:
                    k.fused_bwd_sort(self.pooled, self.small["layout"], ids, offsets, self.B,
                                     self._small_ws(ids.numel()))
            self._barrier(self.site_a)
            k.fused_bwd_sort_peer(self.wire_key, self.wire_idx, self.counts, self.me, self.W, self.cap,
                                  0 if self.bwd_mode == "push" else self.idx_span, g.local.layout, g.overflow,
                                  self._workspace())
            self._prep_pending = True

        self._keep = (ids, offsets, psw)      # the side stream reads them: keep them away from the allocator
        self._on_side(run)

    # ---- backward --------------------------------------------------------------------------------------------------
    def backward(self, grad: torch.Tensor, offsets: torch.Tensor) -> None:
        g, k = self.g, Fn.backend()
        spec = g.local.optimizer
        if spec is None:
            raise RuntimeError("sharded collection: no sparse optimizer set (call set_optimizer)")
        if not self._prep_pending:
            raise RuntimeError("peer exchange: backward without the forward pass's id exchange")
        lay = g.local.layout
        push = self.bwd_mode == "push"
        sm = self.small
        # (TZK_PEER_ACCUM_SIDE=0 switches this off) The per-row sums of the small tables' gradients (a pass over ALL local ids) leave the
        # main stream: they run on the side stream next to the push, followed by a barrier of their own (site_b2) — the
        # main stream only pushes the big tables' rows and crosses barrier B.
        accum_side = (sm is not None and push and os.environ.get("TZK_PEER_ACCUM_SIDE", "1") != "0"
                      and self._side_stream() is not None)
        psw = self._keep[2] if self._keep is not None else None    # this step's weights (prep), or None

        def accumulate_small():
            from .kernels import OPT_ACCUM_OUT

            gr = grad if self.pooled else grad.reshape(-1, g.dim)
            nnz = int(self._keep[0].numel()) if self._keep is not None else 0
            if nnz and psw is not None:     # weighted bags: each entry scaled by (1/W / L) * w before the per-row sums
                k.fused_bwd_apply(OPT_ACCUM_OUT, self.pooled, gr, sm["psum"].t, sm["flags"].t, sm["layout"], offsets, nnz,
                                  self.B, 0.0, 0.0, 1.0 / self.W, self._small_ws(nnz, weighted=True),
                                  per_sample_weights=psw)
            elif nnz:
                k.fused_bwd_apply(OPT_ACCUM_OUT, self.pooled, gr, sm["psum"].t, sm["flags"].t, sm["layout"], offsets, nnz,
                                  self.B, 0.0, 0.0, 1.0 / self.W, self._small_ws(nnz))

        if sm is not None and not accum_side:   # per-row sums of this rank's gradients of the small tables (1/W folded in)
            accumulate_small()
        if accum_side:
            def side_accum():
                accumulate_small()
                self._barrier(self.site_b2)   # every rank's partial sums are complete
            self._on_side(side_accum)         # (forks after everything enqueued so far: the gradient exists)
            # the side stream reads them: away from the allocator until the join
            self._pending_accum = (grad, offsets, psw)
        if push:
            if not self.pooled:
                grad = grad.reshape(-1, g.dim)
            if psw is not None:               # pushed rows are w * g (/ L); wire_w was filled by this step's prep
                k.peer_push_grad(self.recv, grad, lay, offsets, self.wire_idx.t, self.counts.t, self.me, self.W,
                                 self.cap, self.B, self.pooled, wire_w=self.wire_w)
            else:
                k.peer_push_grad(self.recv, grad, lay, offsets, self.wire_idx.t, self.counts.t, self.me, self.W,
                                 self.cap, self.B, self.pooled)
        elif self.pooled:
            ld = g.total_dim
            k.peer_publish_grad(grad, lay, offsets, self.B, self.grad.t.view(self.B, ld))
        else:
            ld = g.dim
            self.grad.t[:grad.numel()].copy_(grad.reshape(-1))
        self._barrier(self.site_b)            # every rank's gradient has arrived / is published
        extras = g.local.opt_extras()

        def run():
            if push:    # the plain sequence-layout update over the local receive buffer (sorted value = its row)
                k.fused_bwd_apply(spec.kind, False, self.recv.t.view(self.W * self.cap, g.dim), g.local.weights.data,
                                  g.local.opt_state, lay, self._dummy_off, self.W * self.cap, 1, spec.lr, spec.eps,
                                  1.0 / self.W, self._workspace(), **extras)
                if sm is not None and sm["total_rows"]:
                    k.peer_small_update(spec.kind, sm["psum"], sm["flags"], self.W, sm["tabs"], sm["n_tabs"],
                                        sm["total_rows"], lay.max_dim, g.local.weights.data, g.local.opt_state, spec.lr,
                                        spec.eps, **extras)
            else:
                k.fused_bwd_apply_peer(spec.kind, self.pooled, self.grad, ld, g.local.weights.data, g.local.opt_state,
                                       lay, self.B, self.me, self.W, self.cap, self.idx_span, spec.lr, spec.eps,
                                       1.0 / self.W, self._workspace(), **extras)
            self._barrier(self.site_c)        # tables quiescent everywhere, wire / receive buffers reusable
            self._prep_pending = False

        self._on_side(run)
        self._keep = None
        self._join_later()

    def _join_later(self) -> None:
        """Joins the side stream when the backward pass ends (the dense backward that autograd still has to run
        overlaps the update); immediately when called outside a backward pass."""
        if self._side_stream() is None:
            return
        cur = torch.cuda.current_stream()

        def join():
            cur.wait_stream(self._side_stream())
            self._pending_accum = None

        if getattr(self, "defer_join", False):    # the step driver joins after the dense optimizer step (join_pending)
            self._pending_join = True
            return
        try:
            torch.autograd.Variable._execution_engine.queue_callback(join)
        except RuntimeError:                  # not inside a backward pass
            join()


def _peer_join_pending(st: "PeerState") -> None:
    if getattr(st, "_pending_join", False) and st._side_stream() is not None:
        torch.cuda.current_stream().wait_stream(st._side_stream())
    st._pending_join = False
    st._pending_accum = None


PeerState.join_pending = _peer_join_pending


class _PeerLookup(torch.autograd.Function):
    """psw: the KJT's per-sample weights (weighted bags) or None; data, no gradient flows to them."""

    @staticmethod
    def forward(ctx, hook, st: PeerState, ids, offsets, psw=None, B=None):
        out = st.gather(ids, offsets, psw, B)
        ctx.st = None
        if hook is not None:                  # (also with zero local ids: the barriers are collective)
            st.prep(ids, offsets, psw)
            ctx.st = st
            ctx.save_for_backward(offsets)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.st is not None:
            (offsets,) = ctx.saved_tensors
            ctx.st.backward(Fn._rows_contig(grad_out) if ctx.st.pooled else grad_out.contiguous(), offsets)
        return None, None, None, None, None, None


def enable_peer_exchange(sm, batch_size: int, ids_per_feature: Optional[Dict[str, int]] = None) -> List[PeerState]:
    """Switches the sharded collection `sm` to the peer-memory path for local batches of `batch_size` samples.
    `ids_per_feature` (KJT key -> ids per step): the id budget of features with more than one id per bag (sequence
    features: batch_size * sequence_length).  Returns the per-dim-group states (kept alive by the patched forward)."""
    grp = sm._group if sm._group is not None else dist.group.WORLD
    states = []
    for g in sm.groups:
        per_f = None
        if ids_per_feature is not None:
            per_f = [int(ids_per_feature.get(name, batch_size)) for name in g.feature_names]
        states.append(PeerState(g, sm.plan, grp, batch_size, per_f))
    pooled = sm._pooled

    def forward(features):
        # weighted id features: each rank's weights stay with its samples (pooled collections, push transport; the
        # checks are host-side, before any launch)
        psw = features.weights_or_none() if pooled else None
        if psw is not None and states:
            states[0]._weights(psw)
        keys, lens, vals = [], [], []
        out = {}
        for g, st in zip(sm.groups, states):
            kjt = g.local._select(features)
            hook = sm._hook_tensor(kjt.values().device)
            # a training step must have the sized batch (the backward's wire layout); a forward-only step (evaluation)
            # may be shorter, e.g. the last batch of an eval set
            if kjt.stride() > st.B or (kjt.stride() != st.B and hook is not None):
                raise RuntimeError(f"peer exchange was sized for batch {st.B}, got {kjt.stride()}")
            res = _PeerLookup.apply(hook, st, kjt.values(), kjt.offsets(), kjt.weights_or_none() if pooled else None,
                                    kjt.stride())
            if pooled:
                vals.append(res)
                keys += g.embedding_names
                lens += [g.dim] * g.F
            else:
                lpk, lengths, B = kjt.length_per_key(), kjt.lengths(), kjt.stride()
                s = 0
                for f, key in enumerate(g.embedding_names):
                    out[key] = JaggedTensor(res[s:s + lpk[f]], lengths=lengths[f * B:(f + 1) * B])
                    s += lpk[f]
        if not pooled:
            return out
        return KeyedTensor(keys, lens, vals[0] if len(vals) == 1 else torch.cat(vals, dim=1))

    sm.forward = forward
    sm._peer_states = states
    return states


class PeerDenseGradSync(PeerBase):
    """Average of the replicated dense gradients through peer memory (the reference wraps dense params in DDP,
    dist_util.py:164-195): gradients accumulate into one flat local buffer; sync() publishes it, crosses one barrier
    and sums all W published buffers in rank order into the flat buffer again — identical bits on every rank, one copy
    + two small kernels, no NCCL."""

    def __init__(self, params: Sequence[torch.nn.Parameter], group=None, world: Optional[int] = None,
                 rank: Optional[int] = None) -> None:
        self.params = [p for p in params if p.requires_grad]
        dev = self.params[0].device if self.params else "cpu"
        super().__init__(group if (group is not None or world is not None) else dist.group.WORLD, dev, world, rank)
        self.world = self.W
        n = sum(p.numel() for p in self.params)
        self.n = n
        self.flat = torch.zeros(max(n, 1), dtype=torch.float32, device=dev)
        self.pub = self._alloc(max(n, 1), torch.float32)
        self.site = _Site(self)
        self.zero()
        self._host_barrier()

    def zero(self) -> None:
        self.flat.zero_()
        o = 0
        for p in self.params:
            if p.grad is None or p.grad.data_ptr() != self.flat[o:o + p.numel()].data_ptr():
                p.grad = self.flat[o:o + p.numel()].view_as(p)
            o += p.numel()

    def sync(self) -> None:
        if self.W == 1 or self.n == 0:
            return
        self.pub.t.copy_(self.flat)
        self._barrier(self.site)
        Fn.backend().peer_allreduce_mean(self.pub, self.W, self.n, self.flat)
