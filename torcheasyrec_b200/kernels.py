"""Tensor-level wrappers over the tzk C-ABI (include/tzk.h).

`CudaKernels` is the only compute backend the package ships.  It validates device / dtype / contiguity,
allocates outputs and workspaces through torch's caching allocator, passes raw pointers + the current
CUDA stream across the ABI, and raises `TzkError` on any failure.  There is deliberately no CPU
implementation here: host-logic tests inject their own checker backend (tests/oracle_backend.py).
"""

import ctypes
import math
import os
import threading
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from ._lib import TzkError, check, lib

POOL_SUM, POOL_MEAN = 0, 1
OPT_SGD, OPT_ADAGRAD, OPT_ROWWISE_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM = 0, 1, 2, 3, 4
OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB, OPT_LARS_SGD = 5, 6, 7      # the layer-wise adaptive optimizers (_ex entry points)
WD_NONE, WD_L2, WD_DECOUPLE = 0, 1, 2    # row-wise Adagrad weight_decay_mode (tzrec WeightDecayMode)
LARS_ETA = 0.001                         # fbgemm's default trust coefficient (tzrec passes none)
OPT_ACCUM_OUT = 100      # peer-memory step: per-row gradient sums into a dense buffer instead of an update


@dataclass
class FeatureLayout:
    """Host-side description of the keys served by one shard arena (one entry per KJT key).

    Mirrors the "feature descriptor" arrays of include/tzk.h.  `key_base` linearises (table,row) for the
    backward sort; features that share a physical table share w_off / key_base.
    """

    w_off: List[int]
    rows: List[int]
    dim: List[int]
    col: List[int]
    pool: List[int]
    key_base: List[int]
    total_keys: int
    total_dim: int
    arena_elems: int
    # elements between consecutive rows of each key's table: None = dense rows (= dim); `interleaved` = every table row is
    # followed by its element-wise optimizer-state row (stride 2 * dim; tzk_opt_args.interleaved, include/tzk.h)
    stride: Optional[List[int]] = None
    interleaved: bool = False
    d_stride: Optional[torch.Tensor] = None
    # device copies (filled by .to())
    d_w_off: Optional[torch.Tensor] = None
    d_rows: Optional[torch.Tensor] = None
    d_dim: Optional[torch.Tensor] = None
    d_col: Optional[torch.Tensor] = None
    d_pool: Optional[torch.Tensor] = None
    d_key_base: Optional[torch.Tensor] = None

    @property
    def num_features(self) -> int:
        return len(self.dim)

    @property
    def max_dim(self) -> int:
        return max(self.dim) if self.dim else 1

    @property
    def vec_ok(self) -> int:
        return int(all(d % 4 == 0 for d in self.dim) and all(c % 4 == 0 for c in self.col)
                   and all(o % 4 == 0 for o in self.w_off) and all(s % 4 == 0 for s in (self.stride or [])))

    def row_stride(self, f: int) -> int:
        return self.stride[f] if self.stride is not None else self.dim[f]

    def to(self, device) -> "FeatureLayout":
        self.d_w_off = torch.tensor(self.w_off, dtype=torch.int64, device=device)
        self.d_rows = torch.tensor(self.rows, dtype=torch.int64, device=device)
        self.d_dim = torch.tensor(self.dim, dtype=torch.int32, device=device)
        self.d_col = torch.tensor(self.col, dtype=torch.int32, device=device)
        self.d_pool = torch.tensor(self.pool, dtype=torch.int32, device=device)
        self.d_key_base = torch.tensor(self.key_base, dtype=torch.int64, device=device)
        self.d_stride = None if self.stride is None else torch.tensor(self.stride, dtype=torch.int32, device=device)
        return self


def build_layout(table_rows: Sequence[int], table_dim: Sequence[int], feat_table: Sequence[int],
                 feat_pool: Sequence[int], align: int = 4, interleaved: bool = False) -> FeatureLayout:
    """Packs tables back to back into one arena (row starts 16-B aligned) and lays features out in order.
    `interleaved`: every table row is followed by its optimizer-state row (row stride 2 * dim; table starts 128-B
    aligned so that a D = 16 row and its state share one line)."""
    t_off, t_key = [], []
    o = k = 0
    mult = 2 if interleaved else 1
    if interleaved:
        align = max(align, 32)
    for r, d in zip(table_rows, table_dim):
        o = (o + align - 1) // align * align
        t_off.append(o)
        t_key.append(k)
        o += r * d * mult
        k += r
    col, c = [], 0
    for t in feat_table:
        col.append(c)
        c += table_dim[t]
    return FeatureLayout(
        w_off=[t_off[t] for t in feat_table], rows=[table_rows[t] for t in feat_table],
        dim=[table_dim[t] for t in feat_table], col=col, pool=list(feat_pool),
        key_base=[t_key[t] for t in feat_table], total_keys=max(k, 1), total_dim=c,
        arena_elems=max(o, 128),   # never smaller than one (widest) row: padding slots read row 0
        stride=[table_dim[t] * 2 for t in feat_table] if interleaved else None, interleaved=interleaved)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    return t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise TzkError(f"{name}: expected a CUDA tensor, got {t.device} (no CPU fallback in torcheasyrec_b200)")
    if t.dtype != dtype:
        raise TzkError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise TzkError(f"{name}: expected a contiguous tensor")
    return t


def _rows2d(t: torch.Tensor, name: str) -> Tuple[torch.Tensor, int]:
    """Accepts a 2-D fp32 CUDA tensor whose rows are contiguous (column slices of a wider buffer are fine)."""
    if not t.is_cuda:
        raise TzkError(f"{name}: expected a CUDA tensor (no CPU fallback)")
    if t.dtype != torch.float32 or t.dim() != 2:
        raise TzkError(f"{name}: expected a 2-D float32 tensor")
    if t.shape[1] > 1 and t.stride(1) != 1:
        raise TzkError(f"{name}: rows must be contiguous")
    ld = t.stride(0) if t.shape[0] > 1 else max(t.shape[1], 1)
    return t, ld


def _rows2d_dtype(t: torch.Tensor, dtype, name: str) -> Tuple[torch.Tensor, int]:
    """_rows2d for another element type (the bf16 interaction's operands)."""
    if not t.is_cuda:
        raise TzkError(f"{name}: expected a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype or t.dim() != 2:
        raise TzkError(f"{name}: expected a 2-D {dtype} tensor")
    if t.shape[1] > 1 and t.stride(1) != 1:
        raise TzkError(f"{name}: rows must be contiguous")
    return t, (t.stride(0) if t.shape[0] > 1 else max(t.shape[1], 1))


def _unvalidated_switch(name: str) -> bool:
    """Mirrors unvalidated_switch() of csrc/tzk_common.cuh: `name`=0/1 decides, else TZK_EXPERIMENTAL=1 turns it on."""
    e = os.environ.get(name, "")
    if e[:1] in ("0", "1"):
        return e[:1] == "1"
    return os.environ.get("TZK_EXPERIMENTAL", "")[:1] == "1"


def _small_linear_rows_path(K: int, N: int) -> bool:
    """Mirrors use_bwd2() of csrc/tzk_tower.cu (launch accounting only)."""
    if os.environ.get("TZK_SMALL_LINEAR_BWD", "")[:1] == "1" or not (1 <= K <= 64 and 1 <= N <= 64):
        return False
    if os.environ.get("TZK_SMALL_LINEAR_DW", "1")[:1] != "0":
        return True
    nb = 4 if N % 4 == 0 else 1
    t = -(-N // nb) * -(-K // 4)
    if t > 128:
        t = -(-N // nb) * -(-K // 8)
    return t <= 128


def norm_family(optimizer: int, ex: dict) -> bool:
    """Mirrors norm_family() of csrc/tzk_bwd.cu: the updates with a norm over the row, which run on the general path."""
    return optimizer in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB, OPT_LARS_SGD) or (
        optimizer == OPT_ROWWISE_ADAGRAD and int(ex.get("weight_decay_mode", WD_NONE)) != WD_NONE
        and float(ex.get("weight_decay", 0.0)) != 0.0)


def _tile_path(lay: "FeatureLayout", optimizer: int = OPT_SGD, ex: Optional[dict] = None) -> bool:
    import os

    return (os.environ.get("TZK_BWD_TILE", "0") == "1" and bool(lay.vec_ok) and lay.max_dim <= 128 and not lay.interleaved
            and not norm_family(optimizer, ex or {}) and (ex or {}).get("per_sample_weights") is None)


def _table_dtype(weights: torch.Tensor, name: str = "weights") -> bool:
    """Validates a table arena (fp32, or fp16 for DataType.FP16 tables); returns True for halfs."""
    if not weights.is_cuda:
        raise TzkError(f"{name}: expected a CUDA tensor, got {weights.device} (no CPU fallback in torcheasyrec_b200)")
    if weights.dtype not in (torch.float32, torch.float16):
        raise TzkError(f"{name}: expected float32 or float16 tables, got {weights.dtype}")
    if not weights.is_contiguous():
        raise TzkError(f"{name}: expected a contiguous tensor")
    return weights.dtype == torch.float16


def _opt_args(optimizer: int, state, lr: float, eps: float, ex: dict):
    """tzk_opt_args (include/tzk.h) for the _ex entry points; keeps the tensors it points to alive via the caller."""
    from ._lib import TzkOptArgs

    st2, step = ex.get("state2"), ex.get("step")
    if optimizer in (OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM, OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB) and (st2 is None or step is None):
        raise TzkError("Adam and LAMB variants need state2 and the device step counter")
    for t, nm in ((st2, "state2"), (step, "step")):
        if t is not None:
            _need(t, torch.float32, nm)
    psw = ex.get("per_sample_weights")
    if psw is not None:
        _need(psw, torch.float32, "per_sample_weights")
    return TzkOptArgs(optimizer, lr, eps, float(ex.get("beta1", 0.9)), float(ex.get("beta2", 0.999)),
                      float(ex.get("weight_decay", 0.0)), float(ex.get("max_gradient", 0.0)),
                      _ptr(state), _ptr(st2), _ptr(step), int(bool(ex.get("weights_f16", False))),
                      int(bool(ex.get("interleaved", False))), float(ex.get("momentum", 0.9)),
                      float(ex.get("eta", LARS_ETA)), int(ex.get("weight_decay_mode", WD_NONE)), _ptr(psw))


class CudaKernels:
    """sm_100a implementation of the hot path.  Stateless apart from cached workspaces."""

    name = "cuda"

    def __init__(self) -> None:
        self._lib = lib()
        self._ws = {}
        self.launches = 0  # hand-written tzk kernels enqueued so far (CUB's sort kernels are not counted)

    # ------------------------------------------------------------------ workspace cache
    def _workspace(self, key, nbytes: int, device) -> torch.Tensor:
        # (per host thread: two threads driving two streams must not share scratch memory)
        slot = (key, device, threading.get_ident())
        ws = self._ws.get(slot)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)
            self._ws[slot] = ws
        return ws

    # ------------------------------------------------------------------ K3
    def lengths_to_offsets(self, lengths: torch.Tensor) -> torch.Tensor:
        _need(lengths, torch.int32, "lengths")
        n = lengths.numel()
        out = torch.empty(n + 1, dtype=torch.int64, device=lengths.device)
        nb = self._lib.tzk_lengths_to_offsets_workspace_bytes(n)
        ws = self._workspace("scan", nb, lengths.device)
        check(self._lib.tzk_lengths_to_offsets(_ptr(lengths), n, _ptr(out), _ptr(ws), ws.numel(), _stream()),
              "tzk_lengths_to_offsets")
        self.launches += 3 if n else 1
        return out

    # ------------------------------------------------------------------ K4
    def pooled_gather_fwd(self, weights: torch.Tensor, lay: FeatureLayout, ids: torch.Tensor,
                          offsets: torch.Tensor, B: int, out: Optional[torch.Tensor] = None,
                          per_sample_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """per_sample_weights (fp32 [nnz], nullable): weighted bags, out = pool_l w[l] * row(ids[l])."""
        f16 = _table_dtype(weights)
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        F = lay.num_features
        if offsets.numel() != F * B + 1:
            raise TzkError(f"offsets has {offsets.numel()} entries, expected F*B+1 = {F * B + 1}")
        if out is None:
            out = torch.empty((B, lay.total_dim), dtype=torch.float32, device=weights.device)
        out, ld = _rows2d(out, "out")
        if per_sample_weights is not None:
            _need(per_sample_weights, torch.float32, "per_sample_weights")
            if per_sample_weights.numel() != ids.numel():
                raise TzkError(f"per_sample_weights has {per_sample_weights.numel()} entries, ids {ids.numel()}")
            if f16 and lay.stride is not None:
                raise TzkError("strided (interleaved) tables are fp32")
            check(self._lib.tzk_pooled_gather_fwd_weighted(
                _ptr(weights), int(f16), _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(lay.d_dim), _ptr(lay.d_stride),
                _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(ids), _ptr(offsets), _ptr(per_sample_weights), F, B,
                lay.max_dim, lay.vec_ok, _ptr(out), ld, _stream()), "tzk_pooled_gather_fwd_weighted")
            self.launches += 1
            return out
        if lay.stride is not None:
            if f16:
                raise TzkError("strided (interleaved) tables are fp32")
            check(self._lib.tzk_pooled_gather_fwd_strided(
                _ptr(weights), _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(lay.d_dim), _ptr(lay.d_stride),
                _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(ids), _ptr(offsets), F, B, lay.max_dim, lay.vec_ok,
                _ptr(out), ld, _stream()), "tzk_pooled_gather_fwd_strided")
            self.launches += 1
            return out
        fn = self._lib.tzk_pooled_gather_fwd_f16 if f16 else self._lib.tzk_pooled_gather_fwd
        check(fn(
            _ptr(weights), _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(lay.d_dim), _ptr(lay.d_col),
            _ptr(lay.d_pool), _ptr(ids), _ptr(offsets), F, B, lay.max_dim, lay.vec_ok, _ptr(out), ld,
            _stream()), "tzk_pooled_gather_fwd")
        self.launches += 1
        return out

    def seq_gather_fwd(self, weights: torch.Tensor, lay: FeatureLayout, ids: torch.Tensor,
                       offsets: torch.Tensor, B: int) -> torch.Tensor:
        f16 = _table_dtype(weights)
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        F = lay.num_features
        D = lay.dim[0] if F else 1
        if any(d != D for d in lay.dim):
            raise TzkError("seq_gather_fwd: all features of an un-pooled collection must share one dim")
        nnz = ids.numel()
        out = torch.empty((nnz, D), dtype=torch.float32, device=weights.device)
        if lay.stride is not None:
            if f16:
                raise TzkError("strided (interleaved) tables are fp32")
            check(self._lib.tzk_seq_gather_fwd_strided(_ptr(weights), _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(ids),
                                                       _ptr(offsets), F, B, D, lay.stride[0] if F else D, nnz, _ptr(out),
                                                       _stream()), "tzk_seq_gather_fwd_strided")
            self.launches += 1
            return out
        fn = self._lib.tzk_seq_gather_fwd_f16 if f16 else self._lib.tzk_seq_gather_fwd
        check(fn(_ptr(weights), _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(ids), _ptr(offsets), F, B, D, nnz, _ptr(out),
                 _stream()), "tzk_seq_gather_fwd")
        self.launches += 1
        return out

    # ------------------------------------------------------------------ K5
    def fused_bwd(self, optimizer: int, pooled: bool, grad_out: torch.Tensor, weights: torch.Tensor,
                  state: Optional[torch.Tensor], lay: FeatureLayout, ids: torch.Tensor, offsets: torch.Tensor,
                  B: int, lr: float, eps: float, grad_scale: float = 1.0, **ex) -> None:
        """`ex` (optional): state2, step, beta1, beta2, weight_decay, max_gradient, momentum, eta, weight_decay_mode,
        per_sample_weights (weighted bags, fp32 [nnz]) -> tzk_fused_bwd_ex."""
        psw = ex.get("per_sample_weights")
        if psw is not None and psw.numel() != ids.numel():
            raise TzkError(f"per_sample_weights has {psw.numel()} entries, ids {ids.numel()}")
        if _table_dtype(weights):
            ex = dict(ex, weights_f16=True)
        if lay.interleaved:
            ex, state = dict(ex, interleaved=True), None    # the state rows live inside `weights`
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        grad_out, ld = _rows2d(grad_out, "grad_out")
        if state is not None:
            _need(state, torch.float32, "state")
        F = lay.num_features
        nnz = ids.numel()
        nb = self.fused_bwd_workspace_bytes(lay, nnz, weighted=psw is not None)
        ws = self._workspace("bwd", nb, weights.device)
        if ex:
            oa = _opt_args(optimizer, state, lr, eps, ex)
            check(self._lib.tzk_fused_bwd_ex(
                ctypes.byref(oa), int(pooled), _ptr(grad_out), ld, _ptr(lay.d_w_off), _ptr(lay.d_rows),
                _ptr(lay.d_dim), _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(lay.d_key_base), _ptr(ids), _ptr(offsets),
                F, B, nnz, lay.total_keys, lay.max_dim, lay.vec_ok, _ptr(weights), grad_scale, _ptr(ws), ws.numel(),
                _stream()), "tzk_fused_bwd_ex")
        else:
            check(self._lib.tzk_fused_bwd(
                optimizer, int(pooled), _ptr(grad_out), ld, _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(lay.d_dim),
                _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(lay.d_key_base), _ptr(ids), _ptr(offsets), F, B, nnz,
                lay.total_keys, lay.max_dim, lay.vec_ok, _ptr(weights), _ptr(state), lr, eps, grad_scale,
                _ptr(ws), ws.numel(), _stream()), "tzk_fused_bwd")
        # own launches next to CUB's radix sort: linearize, zero_counters, find_long_runs (+ sorted_bag_weight for
        # weighted bags) + the gradient half: fused_apply (short runs and the long-run chunk CTAs in ONE launch), or
        # tile_update + carry_combine
        self.launches += (5 if _tile_path(lay, optimizer, ex) else 4) + (psw is not None)

    def fused_bwd_workspace_bytes(self, lay: FeatureLayout, nnz: int, weighted: bool = False) -> int:
        fn = self._lib.tzk_fused_bwd_weighted_workspace_bytes if weighted else self._lib.tzk_fused_bwd_workspace_bytes
        return int(fn(nnz, lay.total_keys, lay.max_dim))

    def fused_bwd_sort(self, pooled: bool, lay: FeatureLayout, ids: torch.Tensor, offsets: torch.Tensor, B: int,
                       ws: torch.Tensor, per_sample_weights: Optional[torch.Tensor] = None) -> None:
        """First half of fused_bwd (linearize + radix sort of (table,row) keys): needs only the ids, so callers run
        it on a side stream while the forward pass is still going.  `ws` must stay untouched until fused_bwd_apply.
        per_sample_weights: weighted bags (tzk_fused_bwd_sort_weighted); the apply then gets the same tensor."""
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        nnz = ids.numel()
        psw = per_sample_weights
        if ws.numel() < self.fused_bwd_workspace_bytes(lay, nnz, weighted=psw is not None):
            raise TzkError("fused_bwd_sort: workspace too small")
        if psw is not None:
            _need(psw, torch.float32, "per_sample_weights")
            if psw.numel() != nnz:
                raise TzkError(f"per_sample_weights has {psw.numel()} entries, ids {nnz}")
            check(self._lib.tzk_fused_bwd_sort_weighted(
                int(pooled), _ptr(lay.d_rows), _ptr(lay.d_key_base), _ptr(ids), _ptr(offsets), _ptr(psw),
                lay.num_features, B, nnz, lay.total_keys, lay.max_dim, _ptr(ws), ws.numel(), _stream()),
                "tzk_fused_bwd_sort_weighted")
            self.launches += 4
            return
        check(self._lib.tzk_fused_bwd_sort(int(pooled), _ptr(lay.d_rows), _ptr(lay.d_key_base), _ptr(ids),
                                           _ptr(offsets), lay.num_features, B, nnz, lay.total_keys, lay.max_dim,
                                           _ptr(ws), ws.numel(), _stream()), "tzk_fused_bwd_sort")
        self.launches += 3

    def fused_bwd_apply(self, optimizer: int, pooled: bool, grad_out: torch.Tensor, weights: torch.Tensor,
                        state: Optional[torch.Tensor], lay: FeatureLayout, offsets: torch.Tensor, nnz: int, B: int,
                        lr: float, eps: float, grad_scale: float, ws: torch.Tensor, **ex) -> None:
        if _table_dtype(weights):
            ex = dict(ex, weights_f16=True)
        if lay.interleaved:
            ex, state = dict(ex, interleaved=True), None    # the state rows live inside `weights`
        _need(offsets, torch.int64, "offsets")
        grad_out, ld = _rows2d(grad_out, "grad_out")
        if optimizer == OPT_ACCUM_OUT:
            _need(state, torch.int32, "state (row flags)")
            ex = dict(ex, max_gradient=0.0)             # -> the _ex entry point
        elif state is not None:
            _need(state, torch.float32, "state")
        if ex:
            oa = _opt_args(optimizer, state, lr, eps, ex)
            check(self._lib.tzk_fused_bwd_apply_ex(
                ctypes.byref(oa), int(pooled), _ptr(grad_out), ld, _ptr(lay.d_w_off), _ptr(lay.d_rows),
                _ptr(lay.d_dim), _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(lay.d_key_base), _ptr(offsets),
                lay.num_features, B, nnz, lay.total_keys, lay.max_dim, lay.vec_ok, _ptr(weights), grad_scale,
                _ptr(ws), ws.numel(), _stream()), "tzk_fused_bwd_apply_ex")
        else:
            check(self._lib.tzk_fused_bwd_apply(
                optimizer, int(pooled), _ptr(grad_out), ld, _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(lay.d_dim),
                _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(lay.d_key_base), _ptr(offsets), lay.num_features, B, nnz,
                lay.total_keys, lay.max_dim, lay.vec_ok, _ptr(weights), _ptr(state), lr, eps, grad_scale,
                _ptr(ws), ws.numel(), _stream()), "tzk_fused_bwd_apply")
        self.launches += 2 if _tile_path(lay, optimizer, ex) else 1

    # ------------------------------------------------------------------ K1 / K2
    def bucketize_rw(self, ids: torch.Tensor, offsets: torch.Tensor, F: int, B: int, W: int,
                     feat_block: torch.Tensor, want_pos: bool = False, feat_owner: Optional[torch.Tensor] = None,
                     want_inv: bool = False, wire_capacity: int = 0):
        """-> (out_lengths [W*F*B], out_offsets [W*F*B+1], out_ids [nnz], out_pos|None, out_inv|None).
        wire_capacity = C > 0: out_ids / out_pos have W*C slots (zero-filled), destination r starts at r*C."""
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        _need(feat_block, torch.int64, "feat_block")
        if feat_owner is not None:
            _need(feat_owner, torch.int32, "feat_owner")
        dev = offsets.device
        nnz = ids.numel()
        out_lengths = torch.empty(W * F * B, dtype=torch.int32, device=dev)
        out_offsets = torch.empty(W * F * B + 1, dtype=torch.int64, device=dev)
        n_out = W * wire_capacity if wire_capacity else nnz
        out_ids = (torch.zeros if wire_capacity else torch.empty)(n_out, dtype=torch.int64, device=dev)
        out_pos = (torch.zeros if wire_capacity else torch.empty)(n_out, dtype=torch.int32, device=dev) \
            if want_pos else None
        out_inv = torch.empty(nnz, dtype=torch.int32, device=dev) if want_inv else None
        nb = self._lib.tzk_bucketize_rw_workspace_bytes(F, B, W, nnz)
        ws = self._workspace("bucketize", nb, dev)
        check(self._lib.tzk_bucketize_rw(_ptr(ids), _ptr(offsets), F, B, W, _ptr(feat_block), _ptr(feat_owner), nnz,
                                         wire_capacity, _ptr(out_lengths), _ptr(out_offsets), _ptr(out_ids), _ptr(out_pos),
                                         _ptr(out_inv), _ptr(ws), ws.numel(), _stream()), "tzk_bucketize_rw")
        self.launches += 5
        return out_lengths, out_offsets, out_ids, out_pos, out_inv

    def bag_grad_expand(self, grad_out: torch.Tensor, lay: FeatureLayout, offsets: torch.Tensor, slot: torch.Tensor,
                        B: int, n_rows: int, zero: bool = False) -> torch.Tensor:
        """g_rows[slot[l]] = grad_out[b, col_f:+D] (/L for MEAN) for every id position l of bag (f,b)."""
        grad_out, ld = _rows2d(grad_out, "grad_out")
        _need(offsets, torch.int64, "offsets")
        _need(slot, torch.int32, "slot")
        D = lay.dim[0]
        if any(d != D for d in lay.dim):
            raise TzkError("bag_grad_expand: all features must share one dim")
        out = (torch.zeros if zero else torch.empty)((n_rows, D), dtype=torch.float32, device=grad_out.device)
        check(self._lib.tzk_bag_grad_expand(_ptr(grad_out), ld, _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(offsets),
                                            _ptr(slot), lay.num_features, B, D, _ptr(out), _stream()),
              "tzk_bag_grad_expand")
        self.launches += 1
        return out

    def permute_lengths(self, lengths: torch.Tensor, perm: torch.Tensor, B: int) -> torch.Tensor:
        _need(lengths, torch.int32, "lengths")
        _need(perm, torch.int32, "perm")
        S = perm.numel()
        out = torch.empty(S * B, dtype=torch.int32, device=lengths.device)
        check(self._lib.tzk_permute_lengths(_ptr(lengths), _ptr(perm), S, B, _ptr(out), _stream()),
              "tzk_permute_lengths")
        self.launches += 1
        return out

    def permute_ids(self, ids: torch.Tensor, in_offsets: torch.Tensor, out_offsets: torch.Tensor,
                    perm: torch.Tensor, B: int, out_nnz: int) -> torch.Tensor:
        _need(ids, torch.int64, "ids")
        _need(in_offsets, torch.int64, "in_offsets")
        _need(out_offsets, torch.int64, "out_offsets")
        _need(perm, torch.int32, "perm")
        out = torch.empty(out_nnz, dtype=torch.int64, device=ids.device)
        check(self._lib.tzk_permute_ids(_ptr(ids), _ptr(in_offsets), _ptr(out_offsets), _ptr(perm),
                                        perm.numel(), B, _ptr(out), _stream()), "tzk_permute_ids")
        self.launches += 1
        return out

    def permute_weights(self, weights: torch.Tensor, in_offsets: torch.Tensor, out_offsets: torch.Tensor,
                        perm: torch.Tensor, B: int, out_nnz: int) -> torch.Tensor:
        """The per-sample weights of a weighted KJT, moved like its ids (permute_ids)."""
        _need(weights, torch.float32, "weights")
        _need(in_offsets, torch.int64, "in_offsets")
        _need(out_offsets, torch.int64, "out_offsets")
        _need(perm, torch.int32, "perm")
        out = torch.empty(out_nnz, dtype=torch.float32, device=weights.device)
        check(self._lib.tzk_permute_weights(_ptr(weights), _ptr(in_offsets), _ptr(out_offsets), _ptr(perm),
                                            perm.numel(), B, _ptr(out), _stream()), "tzk_permute_weights")
        self.launches += 1
        return out

    # ------------------------------------------------------------------ DIN attention over jagged rows (tzk_din.cu)
    def din_attn_input_fwd(self, query: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
        query, ld_q = _rows2d(query, "query")
        _need(seq, torch.float32, "seq")
        _need(offsets, torch.int64, "offsets")
        B, Dq = query.shape
        N, Ds = seq.shape
        out = torch.empty((N, 4 * Ds), dtype=torch.float32, device=seq.device)
        check(self._lib.tzk_din_attn_input_fwd(_ptr(query), ld_q, Dq, _ptr(seq), _ptr(offsets), B, Ds, N, _ptr(out),
                                               _stream()), "tzk_din_attn_input_fwd")
        self.launches += 1 if N else 0
        return out

    def din_attn_input_bwd(self, d_in: torch.Tensor, query: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor):
        query, ld_q = _rows2d(query, "query")
        _need(d_in, torch.float32, "d_in")
        _need(seq, torch.float32, "seq")
        B, Dq = query.shape
        N, Ds = seq.shape
        d_query = torch.empty((B, Dq), dtype=torch.float32, device=seq.device)
        d_seq = torch.empty((N, Ds), dtype=torch.float32, device=seq.device)
        check(self._lib.tzk_din_attn_input_bwd(_ptr(d_in), _ptr(query), ld_q, Dq, _ptr(seq), _ptr(offsets), B, Ds, N,
                                               _ptr(d_query), _ptr(d_seq), _stream()), "tzk_din_attn_input_bwd")
        self.launches += 1
        return d_query, d_seq

    def jagged_softmax_wsum_fwd(self, scores: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor, max_len: int = 0):
        _need(scores, torch.float32, "scores")
        _need(seq, torch.float32, "seq")
        _need(offsets, torch.int64, "offsets")
        N, Ds = seq.shape
        B = offsets.numel() - 1
        probs = torch.empty(N, dtype=torch.float32, device=seq.device)
        out = torch.empty((B, Ds), dtype=torch.float32, device=seq.device)
        check(self._lib.tzk_jagged_softmax_wsum_fwd(_ptr(scores), _ptr(seq), _ptr(offsets), B, Ds, int(max_len), N,
                                                    _ptr(probs), _ptr(out), _stream()), "tzk_jagged_softmax_wsum_fwd")
        self.launches += 1
        return probs, out

    def jagged_softmax_wsum_bwd(self, d_out: torch.Tensor, probs: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor,
                                max_len: int = 0):
        _need(d_out, torch.float32, "d_out")
        _need(probs, torch.float32, "probs")
        N, Ds = seq.shape
        B = offsets.numel() - 1
        d_scores = torch.empty(N, dtype=torch.float32, device=seq.device)
        d_seq = torch.empty((N, Ds), dtype=torch.float32, device=seq.device)
        check(self._lib.tzk_jagged_softmax_wsum_bwd(_ptr(d_out), _ptr(probs), _ptr(seq), _ptr(offsets), B, Ds,
                                                    int(max_len), N, _ptr(d_scores), _ptr(d_seq), _stream()),
              "tzk_jagged_softmax_wsum_bwd")
        self.launches += 1 if N else 0
        return d_scores, d_seq

    # ------------------------------------------------------------------ sharded step over peer memory (tzk_peer.cu)
    # `symm` arguments: objects with `.ptrs` = ctypes array [W] of device addresses (rank r's symmetric buffer as
    # mapped in this process) — peer_exchange._Symm.  The table arenas' `.t` says their element type: float32, or float16
    # for FP16 tables (the _f16 entry points; the mirror then holds halfs too).
    @staticmethod
    def _peer_f16(tables, mirror: Optional[torch.Tensor]) -> bool:
        t = getattr(tables, "t", None)
        dt = torch.float32 if t is None else t.dtype
        if dt not in (torch.float32, torch.float16):
            raise TzkError(f"peer tables: expected float32 or float16 arenas, got {dt}")
        if mirror is not None:
            _need(mirror, dt, "mirror")
        return dt == torch.float16

    def peer_pooled_gather_fwd(self, tables, rf_w_off: torch.Tensor, feat_rows: torch.Tensor, feat_block: torch.Tensor,
                               feat_owner: torch.Tensor, lay: FeatureLayout, ids: torch.Tensor, offsets: torch.Tensor,
                               B: int, W: int, out: Optional[torch.Tensor] = None, mirror: Optional[torch.Tensor] = None,
                               feat_mirror_off: Optional[torch.Tensor] = None,
                               feat_sel: Optional[torch.Tensor] = None,
                               per_sample_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`feat_sel` (device int32 indices): serve only these features (their output columns); `out` is then required.
        `per_sample_weights` (fp32 [nnz], nullable): weighted bags, pooled as pooled_gather_fwd pools them."""
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        f16 = self._peer_f16(tables, mirror)
        F = lay.num_features
        if offsets.numel() != F * B + 1:
            raise TzkError(f"offsets has {offsets.numel()} entries, expected F*B+1 = {F * B + 1}")
        if not lay.vec_ok:
            raise TzkError("peer gather: rows must be 16-B aligned (dims and offsets multiples of 4 floats)")
        if out is None:
            out = torch.empty((B, lay.total_dim), dtype=torch.float32, device=ids.device)
        out, ld = _rows2d(out, "out")
        psw = per_sample_weights
        if psw is not None and ids.numel():      # (no ids: every bag is empty, the unweighted launch writes the zeros)
            _need(psw, torch.float32, "per_sample_weights")
            if psw.numel() != ids.numel():
                raise TzkError(f"per_sample_weights has {psw.numel()} entries, ids {ids.numel()}")
            if feat_sel is not None:
                _need(feat_sel, torch.int32, "feat_sel")
            fn = (self._lib.tzk_peer_pooled_gather_fwd_weighted_f16 if f16
                  else self._lib.tzk_peer_pooled_gather_fwd_weighted)
            check(fn(
                tables.ptrs, _ptr(rf_w_off), _ptr(feat_rows), _ptr(feat_block), _ptr(feat_owner), _ptr(lay.d_dim),
                _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(ids), _ptr(offsets), F, B, W, (lay.max_dim + 3) // 4 * 4,
                _ptr(out), ld, _ptr(mirror), _ptr(feat_mirror_off), _ptr(psw), _ptr(feat_sel),
                0 if feat_sel is None else feat_sel.numel(), _stream()), "tzk_peer_pooled_gather_fwd_weighted")
            self.launches += 1
            return out
        if feat_sel is not None:
            _need(feat_sel, torch.int32, "feat_sel")
            fn = self._lib.tzk_peer_pooled_gather_fwd_sel_f16 if f16 else self._lib.tzk_peer_pooled_gather_fwd_sel
            check(fn(
                tables.ptrs, _ptr(rf_w_off), _ptr(feat_rows), _ptr(feat_block), _ptr(feat_owner), _ptr(lay.d_dim),
                _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(ids), _ptr(offsets), F, B, W, (lay.max_dim + 3) // 4 * 4,
                _ptr(out), ld, _ptr(mirror), _ptr(feat_mirror_off), _ptr(feat_sel), feat_sel.numel(), _stream()),
                "tzk_peer_pooled_gather_fwd_sel")
            self.launches += 1
            return out
        fn = self._lib.tzk_peer_pooled_gather_fwd_f16 if f16 else self._lib.tzk_peer_pooled_gather_fwd
        check(fn(
            tables.ptrs, _ptr(rf_w_off), _ptr(feat_rows), _ptr(feat_block), _ptr(feat_owner), _ptr(lay.d_dim),
            _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(ids), _ptr(offsets), F, B, W, (lay.max_dim + 3) // 4 * 4, _ptr(out),
            ld, _ptr(mirror), _ptr(feat_mirror_off), _stream()), "tzk_peer_pooled_gather_fwd")
        self.launches += 1
        return out

    def peer_seq_gather_fwd(self, tables, rf_w_off: torch.Tensor, feat_rows: torch.Tensor, feat_block: torch.Tensor,
                            feat_owner: torch.Tensor, lay: FeatureLayout, ids: torch.Tensor, offsets: torch.Tensor,
                            B: int, W: int, mirror: Optional[torch.Tensor] = None,
                            feat_mirror_off: Optional[torch.Tensor] = None) -> torch.Tensor:
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        f16 = self._peer_f16(tables, mirror)
        F, D, nnz = lay.num_features, lay.dim[0], ids.numel()
        out = torch.empty((nnz, D), dtype=torch.float32, device=ids.device)
        fn = self._lib.tzk_peer_seq_gather_fwd_f16 if f16 else self._lib.tzk_peer_seq_gather_fwd
        check(fn(tables.ptrs, _ptr(rf_w_off), _ptr(feat_rows), _ptr(feat_block), _ptr(feat_owner), _ptr(ids),
                 _ptr(offsets), F, B, W, D, nnz, _ptr(out), _ptr(mirror), _ptr(feat_mirror_off), _stream()),
              "tzk_peer_seq_gather_fwd")
        self.launches += 1 if nnz else 0
        return out

    def peer_mirror_refresh(self, tables, W: int, seg_rank: torch.Tensor, seg_src: torch.Tensor, seg_dst: torch.Tensor,
                            seg_n: torch.Tensor, mirror: torch.Tensor) -> None:
        """This step's local copy of the small tables (see tzk_peer_mirror_refresh); FP16 tables: a mirror of halfs."""
        f16 = self._peer_f16(tables, mirror)
        fn = self._lib.tzk_peer_mirror_refresh_f16 if f16 else self._lib.tzk_peer_mirror_refresh
        check(fn(tables.ptrs, W, _ptr(seg_rank), _ptr(seg_src), _ptr(seg_dst), _ptr(seg_n), seg_rank.numel(), _ptr(mirror),
                 _stream()), "tzk_peer_mirror_refresh")
        self.launches += 1

    def peer_barrier(self, pads, me: int, W: int, epoch: torch.Tensor) -> None:
        check(self._lib.tzk_peer_barrier(pads.ptrs, me, W, _ptr(epoch), _stream()), "tzk_peer_barrier")
        self.launches += 1

    def peer_bucketize(self, ids: torch.Tensor, offsets: torch.Tensor, F: int, B: int, W: int, feat_block: torch.Tensor,
                       feat_owner: torch.Tensor, feat_rows: torch.Tensor, rf_key_base: torch.Tensor, pooled: bool,
                       cap: int, wire_key: torch.Tensor, wire_idx: torch.Tensor, counts: torch.Tensor,
                       per_sample_weights: Optional[torch.Tensor] = None, wire_w: Optional[torch.Tensor] = None) -> None:
        """ids of the local batch -> this rank's own wire buffers (see tzk_peer_bucketize in include/tzk.h).  Weighted
        bags (pooled): `per_sample_weights` [nnz] and `wire_w` (local fp32 [W * cap]) receive every slot's weight."""
        _need(ids, torch.int64, "ids")
        _need(offsets, torch.int64, "offsets")
        _need(wire_key, torch.int64, "wire_key")
        _need(wire_idx, torch.int32, "wire_idx")
        _need(counts, torch.int32, "counts")
        if wire_key.numel() < W * cap or wire_idx.numel() < W * cap or counts.numel() < W + 1:
            raise TzkError("peer_bucketize: wire buffers smaller than W * cap")
        nb = self._lib.tzk_peer_bucketize_workspace_bytes(F, B, W)
        ws = self._workspace(("peer_bkt", F, B, W), nb, ids.device)
        psw = per_sample_weights
        if psw is not None and ids.numel():      # (no ids: no slot is filled, so no weight is read)
            _need(psw, torch.float32, "per_sample_weights")
            if wire_w is None:
                raise TzkError("peer_bucketize: weighted bags need wire_w")
            _need(wire_w, torch.float32, "wire_w")
            if not pooled or psw.numel() != ids.numel() or wire_w.numel() < W * cap:
                raise TzkError("peer_bucketize: per-sample weights need the pooled layout, one weight per id and "
                               "W * cap wire_w entries")
            check(self._lib.tzk_peer_bucketize_weighted(
                _ptr(ids), _ptr(offsets), F, B, W, _ptr(feat_block), _ptr(feat_owner), _ptr(feat_rows),
                _ptr(rf_key_base), int(pooled), cap, _ptr(wire_key), _ptr(wire_idx), _ptr(counts), _ptr(ws), ws.numel(),
                _ptr(psw), _ptr(wire_w), _stream()), "tzk_peer_bucketize_weighted")
            self.launches += 3
            return
        check(self._lib.tzk_peer_bucketize(_ptr(ids), _ptr(offsets), F, B, W, _ptr(feat_block), _ptr(feat_owner),
                                           _ptr(feat_rows), _ptr(rf_key_base), int(pooled), cap, _ptr(wire_key),
                                           _ptr(wire_idx), _ptr(counts), _ptr(ws), ws.numel(), _stream()),
              "tzk_peer_bucketize")
        self.launches += 3

    def peer_publish_grad(self, grad: torch.Tensor, lay: FeatureLayout, offsets: torch.Tensor, B: int,
                          dst: torch.Tensor) -> None:
        grad, ld = _rows2d(grad, "grad")
        dst, ld_dst = _rows2d(dst, "dst")
        if POOL_MEAN not in lay.pool:        # plain copy: no per-bag scale to fold in
            dst.copy_(grad)
            return
        check(self._lib.tzk_peer_publish_grad(_ptr(grad), ld, _ptr(lay.d_col), _ptr(lay.d_dim), _ptr(lay.d_pool),
                                              _ptr(offsets), lay.num_features, B, _ptr(dst), ld_dst, _stream()),
              "tzk_peer_publish_grad")
        self.launches += 1

    def peer_push_grad(self, recv, grad: torch.Tensor, lay: FeatureLayout, offsets: torch.Tensor, wire_idx: torch.Tensor,
                       counts: torch.Tensor, me: int, W: int, cap: int, B: int, pooled: bool,
                       wire_w: Optional[torch.Tensor] = None) -> None:
        """This rank's gradient slices -> the owners' receive buffers, wire order (see tzk_peer_push_grad).  `wire_w`
        (weighted bags, pooled; filled by peer_bucketize): every slice is pushed as w * g (/ L)."""
        grad, ld = _rows2d(grad, "grad")
        _need(wire_idx, torch.int32, "wire_idx")
        _need(counts, torch.int32, "counts")
        if wire_w is not None:
            _need(wire_w, torch.float32, "wire_w")
            if not pooled or wire_w.numel() < W * cap:
                raise TzkError("peer_push_grad: wire_w needs the pooled layout and W * cap entries")
            check(self._lib.tzk_peer_push_grad_weighted(
                recv.ptrs, _ptr(grad), ld, _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(offsets), _ptr(wire_idx),
                _ptr(counts), me, W, cap, B, lay.dim[0], int(pooled), _ptr(wire_w), _stream()),
                "tzk_peer_push_grad_weighted")
            self.launches += 1
            return
        check(self._lib.tzk_peer_push_grad(recv.ptrs, _ptr(grad), ld, _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(offsets),
                                           _ptr(wire_idx), _ptr(counts), me, W, cap, B, lay.dim[0], int(pooled),
                                           _stream()), "tzk_peer_push_grad")
        self.launches += 1

    def peer_allreduce_mean(self, srcs, W: int, n: int, out: torch.Tensor) -> None:
        _need(out, torch.float32, "out")
        check(self._lib.tzk_peer_allreduce_mean(srcs.ptrs, W, n, _ptr(out), _stream()), "tzk_peer_allreduce_mean")
        self.launches += 1

    def peer_small_update(self, optimizer: int, psum, flags, W: int, tabs: torch.Tensor, n_tabs: int, total_rows: int,
                          max_dim: int, weights: torch.Tensor, state: Optional[torch.Tensor], lr: float, eps: float,
                          **ex) -> None:
        """Owner side of the small-table exchange (see tzk_peer_small_update): psum / flags are symmetric buffers."""
        if _table_dtype(weights):             # FP16 tables: fp32 partial sums, the half row rounded back
            ex = dict(ex, weights_f16=True)
        oa = _opt_args(optimizer, state, lr, eps, ex)
        check(self._lib.tzk_peer_small_update(ctypes.byref(oa), psum.ptrs, flags.ptrs, W, _ptr(tabs), n_tabs, total_rows,
                                              max_dim, _ptr(weights), _stream()), "tzk_peer_small_update")
        self.launches += 1

    def fused_bwd_sort_peer(self, wire_key, wire_idx, counts, me: int, W: int, cap: int, idx_span: int,
                            lay: FeatureLayout, overflow: Optional[torch.Tensor], ws: torch.Tensor) -> None:
        if ws.numel() < self.fused_bwd_workspace_bytes(lay, W * cap):
            raise TzkError("fused_bwd_sort_peer: workspace too small")
        # idx_span == 0: "slot mode" (the gradient rows are pushed to this rank's receive buffer: value = its row)
        check(self._lib.tzk_fused_bwd_sort_peer(wire_key.ptrs, wire_idx.ptrs if idx_span else None, counts.ptrs, me, W,
                                                cap, idx_span,
                                                lay.total_keys, lay.max_dim, _ptr(overflow), _ptr(ws), ws.numel(),
                                                _stream()), "tzk_fused_bwd_sort_peer")
        self.launches += 3

    def fused_bwd_apply_peer(self, optimizer: int, pooled: bool, grads, ld_grad: int, weights: torch.Tensor,
                             state: Optional[torch.Tensor], lay: FeatureLayout, B: int, me: int, W: int, cap: int,
                             idx_span: int, lr: float, eps: float, grad_scale: float, ws: torch.Tensor, **ex) -> None:
        if _table_dtype(weights):             # FP16 tables: the gradients stay fp32, the update rounds the half row
            ex = dict(ex, weights_f16=True)
        if state is not None:
            _need(state, torch.float32, "state")
        oa = _opt_args(optimizer, state, lr, eps, ex)
        check(self._lib.tzk_fused_bwd_apply_peer(
            ctypes.byref(oa), int(pooled), grads.ptrs, ld_grad, _ptr(lay.d_w_off), _ptr(lay.d_rows), _ptr(lay.d_dim),
            _ptr(lay.d_col), _ptr(lay.d_pool), _ptr(lay.d_key_base), lay.num_features, B, me, W, cap, idx_span,
            lay.total_keys, lay.max_dim, lay.vec_ok, _ptr(weights), grad_scale, _ptr(ws), ws.numel(), _stream()),
            "tzk_fused_bwd_apply_peer")
        self.launches += 2 if _tile_path(lay, optimizer, ex) else 1

    # ------------------------------------------------------------------ K6
    def col_gather_sum(self, srcs: Sequence[torch.Tensor], plan: "ColPlan", rows: int,
                       out: Optional[torch.Tensor] = None) -> torch.Tensor:
        lds = []
        for i, s in enumerate(srcs):
            s, ld = _rows2d(s, f"srcs[{i}]")
            lds.append(ld)
        dev = srcs[0].device
        if out is None:
            out = torch.empty((rows, plan.C), dtype=torch.float32, device=dev)
        out, ld_out = _rows2d(out, "out")
        n = len(srcs)
        ptrs = (ctypes.c_void_p * n)(*[s.data_ptr() for s in srcs])  # host arrays -> kernel parameters
        ldt = (ctypes.c_int64 * n)(*lds)
        check(self._lib.tzk_col_gather_sum(ptrs, ldt, n, _ptr(plan.d_col_start), _ptr(plan.d_col_src),
                                           _ptr(plan.d_col_srccol), plan.C, rows, _ptr(out), ld_out, _stream()),
              "tzk_col_gather_sum")
        self.launches += 1
        return out

    # ------------------------------------------------------------------ K7
    def jagged_to_padded(self, values: torch.Tensor, offsets: torch.Tensor, T: int) -> torch.Tensor:
        _need(values, torch.float32, "values")
        _need(offsets, torch.int64, "offsets")
        B = offsets.numel() - 1
        D = values.shape[1]
        out = torch.empty((B, T, D), dtype=torch.float32, device=values.device)
        check(self._lib.tzk_jagged_to_padded(_ptr(values), _ptr(offsets), B, T, D, _ptr(out), _stream()),
              "tzk_jagged_to_padded")
        self.launches += 1
        return out

    def padded_to_jagged(self, grad_out: torch.Tensor, offsets: torch.Tensor, nnz: int) -> torch.Tensor:
        _need(grad_out, torch.float32, "grad_out")
        _need(offsets, torch.int64, "offsets")
        B, T, D = grad_out.shape
        out = torch.empty((nnz, D), dtype=torch.float32, device=grad_out.device)
        check(self._lib.tzk_padded_to_jagged(_ptr(grad_out), _ptr(offsets), B, T, D, nnz, _ptr(out), _stream()),
              "tzk_padded_to_jagged")
        self.launches += 1
        return out

    # ------------------------------------------------------------------ A7
    def fm_fwd(self, x: torch.Tensor, N: int, D: int) -> torch.Tensor:
        x, ld = _rows2d(x, "x")
        B = x.shape[0]
        y = torch.empty((B, D), dtype=torch.float32, device=x.device)
        check(self._lib.tzk_fm_fwd(_ptr(x), ld, B, N, D, _ptr(y), D, _stream()), "tzk_fm_fwd")
        self.launches += 1
        return y

    def fm_bwd(self, x: torch.Tensor, dy: torch.Tensor, N: int, D: int) -> torch.Tensor:
        x, ld = _rows2d(x, "x")
        dy, ld_dy = _rows2d(dy, "dy")
        B = x.shape[0]
        dx = torch.empty((B, N * D), dtype=torch.float32, device=x.device)
        check(self._lib.tzk_fm_bwd(_ptr(x), ld, _ptr(dy), ld_dy, B, N, D, _ptr(dx), N * D, _stream()),
              "tzk_fm_bwd")
        self.launches += 1
        return dx

    # ------------------------------------------------------------------ A9 / A10
    def dot_interact_fwd(self, dense: Optional[torch.Tensor], sparse: torch.Tensor, Ns: int, D: int,
                         copy_dense: bool, copy_sparse: bool, pad_to: int = 1, p_pad: int = 0) -> torch.Tensor:
        """Layout [P | p_pad zeros | dense D | sparse Ns*D | tail zeros up to a multiple of pad_to]."""
        sparse, ld_s = _rows2d(sparse, "sparse")
        B = sparse.shape[0]
        ld_d = 0
        if dense is not None:
            dense, ld_d = _rows2d(dense, "dense")
        N = Ns + (dense is not None)
        width = N * (N - 1) // 2 + p_pad + (D if (copy_dense and dense is not None) else 0) + \
            (Ns * D if copy_sparse else 0)
        wp = (width + pad_to - 1) // pad_to * pad_to
        out = torch.empty((B, wp), dtype=torch.float32, device=sparse.device)
        if wp != width:
            out[:, width:].zero_()
        check(self._lib.tzk_dot_interact_fwd(_ptr(dense), ld_d, _ptr(sparse), ld_s, B, Ns, D, int(copy_dense),
                                             int(copy_sparse), p_pad, _ptr(out), wp, _stream()),
              "tzk_dot_interact_fwd")
        self.launches += 1
        return out

    def dot_interact_bwd(self, dense: Optional[torch.Tensor], sparse: torch.Tensor, d_out: torch.Tensor,
                         Ns: int, D: int, copy_dense: bool, copy_sparse: bool, p_pad: int = 0):
        sparse, ld_s = _rows2d(sparse, "sparse")
        d_out, ld_o = _rows2d(d_out, "d_out")
        B = sparse.shape[0]
        ld_d = 0
        d_dense = None
        if dense is not None:
            dense, ld_d = _rows2d(dense, "dense")
            d_dense = torch.empty((B, D), dtype=torch.float32, device=sparse.device)
        d_sparse = torch.empty((B, Ns * D), dtype=torch.float32, device=sparse.device)
        check(self._lib.tzk_dot_interact_bwd(_ptr(dense), ld_d, _ptr(sparse), ld_s, _ptr(d_out), ld_o, B, Ns, D,
                                             int(copy_dense), int(copy_sparse), p_pad, _ptr(d_dense), D,
                                             _ptr(d_sparse), Ns * D, _stream()), "tzk_dot_interact_bwd")
        self.launches += 1
        return d_dense, d_sparse

    def dot_interact27_fwd_bf16(self, dense: torch.Tensor, sparse: torch.Tensor) -> torch.Tensor:
        """X [B, 784] bf16 = [351 pairs | 0 | dense | bf16(sparse)] of DLRM-Criteo's interaction under bf16 autocast, from
        dense [B, 16] bf16 and sparse [B, 416] fp32 (tzk_dot_interact27_fwd_bf16)."""
        dense, ld_d = _rows2d_dtype(dense, torch.bfloat16, "dense")
        sparse, ld_s = _rows2d(sparse, "sparse")
        B = sparse.shape[0]
        if tuple(dense.shape) != (B, 16) or tuple(sparse.shape) != (B, 416):
            raise TzkError(f"dot_interact27_fwd_bf16: expected dense [B, 16] and sparse [B, 416], got "
                           f"{tuple(dense.shape)} and {tuple(sparse.shape)}")
        out = torch.empty((B, 784), dtype=torch.bfloat16, device=sparse.device)
        check(self._lib.tzk_dot_interact27_fwd_bf16(_ptr(dense), ld_d, _ptr(sparse), ld_s, B, _ptr(out), 784, _stream()),
              "tzk_dot_interact27_fwd_bf16")
        self.launches += 1
        return out

    def dot_interact27_bwd_bf16(self, d_out: torch.Tensor, dense: torch.Tensor, sparse: torch.Tensor):
        """(d_dense [B, 16] bf16, d_sparse [B, 416] fp32) from dX [B, 784] bf16 (tzk_dot_interact27_bwd_bf16)."""
        d_out, ld_o = _rows2d_dtype(d_out, torch.bfloat16, "d_out")
        dense, ld_d = _rows2d_dtype(dense, torch.bfloat16, "dense")
        sparse, ld_s = _rows2d(sparse, "sparse")
        B = sparse.shape[0]
        if tuple(d_out.shape) != (B, 784) or tuple(dense.shape) != (B, 16) or tuple(sparse.shape) != (B, 416):
            raise TzkError(f"dot_interact27_bwd_bf16: expected dX [B, 784], dense [B, 16] and sparse [B, 416], got "
                           f"{tuple(d_out.shape)}, {tuple(dense.shape)} and {tuple(sparse.shape)}")
        d_dense = torch.empty((B, 16), dtype=torch.bfloat16, device=sparse.device)
        d_sparse = torch.empty((B, 416), dtype=torch.float32, device=sparse.device)
        check(self._lib.tzk_dot_interact27_bwd_bf16(_ptr(d_out), ld_o, _ptr(dense), ld_d, _ptr(sparse), ld_s, B,
                                                    _ptr(d_dense), 16, _ptr(d_sparse), 416, _stream()),
              "tzk_dot_interact27_bwd_bf16")
        self.launches += 1
        return d_dense, d_sparse

    def interact_wide_fwd(self, dense: torch.Tensor, sparse: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor]):
        """(y [B, 64], pairs [B, 352]): relu(X w^T + bias) of DLRM-Criteo's interaction output X [B, 784] (never written)
        and X's pair columns, with w [64, 784] in the interaction's column layout."""
        dense, ld_d = _rows2d(dense, "dense")
        sparse, ld_s = _rows2d(sparse, "sparse")
        w, ld_w = _rows2d(w, "w")
        B = dense.shape[0]
        y = torch.empty((B, 64), dtype=torch.float32, device=dense.device)
        pairs = torch.empty((B, 352), dtype=torch.float32, device=dense.device)
        ws = torch.empty((2, 64, 784), dtype=torch.float32, device=dense.device)
        check(self._lib.tzk_interact_wide_fwd(_ptr(dense), ld_d, _ptr(sparse), ld_s, _ptr(w), ld_w, _ptr(bias), B,
                                              _ptr(y), 64, _ptr(pairs), 352, _ptr(ws[0]), _ptr(ws[1]), _stream()),
              "tzk_interact_wide_fwd")
        self.launches += 2
        return y, pairs

    def interact_wide_wgrad(self, dz: torch.Tensor, pairs: torch.Tensor, dense: torch.Tensor, sparse: torch.Tensor,
                            slabs: int, scale: Optional[torch.Tensor] = None) -> torch.Tensor:
        """dW [64, 784] = dz^T X in the interaction's column layout, X = [pairs | dense | sparse] read in place.  `scale`:
        a one-element fp32 tensor on the device; dz is read times it (the bits of passing dz * scale)."""
        dz, ld_z = _rows2d(dz, "dz")
        pairs, ld_p = _rows2d(pairs, "pairs")
        dense, ld_d = _rows2d(dense, "dense")
        sparse, ld_s = _rows2d(sparse, "sparse")
        B = dz.shape[0]
        dw = torch.empty((64, 784), dtype=torch.float32, device=dz.device)
        part = torch.empty(slabs * 896 * 64, dtype=torch.float32, device=dz.device)
        if scale is not None and _need(scale, torch.float32, "scale").numel() != 1:
            raise TzkError("scale: expected one element")
        check(self._lib.tzk_interact_wide_wgrad_scaled(_ptr(dz), ld_z, _ptr(scale), _ptr(pairs), ld_p, _ptr(dense), ld_d,
                                                       _ptr(sparse), ld_s, B, slabs, _ptr(part), _ptr(dw), 784,
                                                       _stream()), "tzk_interact_wide_wgrad_scaled")
        self.launches += 2
        return dw

    def interact_wide_bwd(self, dz: torch.Tensor, w: torch.Tensor, dense: torch.Tensor, sparse: torch.Tensor,
                          scale: Optional[torch.Tensor] = None):
        """(d_dense [B, 16], d_sparse [B, 416]) of DLRM-Criteo's interaction followed by a 784 -> 64 layer with weight
        w [64, 784] (the interaction's column layout), from dz [B, 64], the gradient of the layer's pre-activation.
        `scale`: as in interact_wide_wgrad."""
        dz, ld_z = _rows2d(dz, "dz")
        w, ld_w = _rows2d(w, "w")
        dense, ld_d = _rows2d(dense, "dense")
        sparse, ld_s = _rows2d(sparse, "sparse")
        B = dz.shape[0]
        d_dense = torch.empty((B, 16), dtype=torch.float32, device=dz.device)
        d_sparse = torch.empty((B, 416), dtype=torch.float32, device=dz.device)
        wt = torch.empty((2, 784, 64), dtype=torch.float32, device=dz.device)
        if scale is not None and _need(scale, torch.float32, "scale").numel() != 1:
            raise TzkError("scale: expected one element")
        check(self._lib.tzk_interact_wide_bwd_scaled(_ptr(dz), ld_z, _ptr(scale), _ptr(w), ld_w, _ptr(dense), ld_d,
                                                     _ptr(sparse), ld_s, B, _ptr(d_dense), 16, _ptr(d_sparse), 416,
                                                     _ptr(wt[0]), _ptr(wt[1]), _stream()),
              "tzk_interact_wide_bwd_scaled")
        self.launches += 2
        return d_dense, d_sparse

    # ------------------------------------------------------------------ dense-tower helpers
    def bias_act(self, y: torch.Tensor, bias: Optional[torch.Tensor], relu: bool) -> torch.Tensor:
        y, ld = _rows2d(y, "y")
        check(self._lib.tzk_bias_act(_ptr(y), ld, _ptr(bias), y.shape[0], y.shape[1], int(relu), _stream()),
              "tzk_bias_act")
        self.launches += 1
        return y

    def act_bwd_colsum(self, dy: torch.Tensor, y: Optional[torch.Tensor], relu: bool, want_dz: bool = True,
                       out: Optional[torch.Tensor] = None):
        """`out`: where dz goes (a [M, N] view with contiguous rows, which may be dy itself); None allocates it."""
        dy, ld_dy = _rows2d(dy, "dy")
        M, N = dy.shape
        ld_y = 0
        if y is not None:
            y, ld_y = _rows2d(y, "y")
        if out is not None:
            dz, ld_dz = _rows2d(out, "out")
        else:
            dz, ld_dz = (torch.empty((M, N), dtype=torch.float32, device=dy.device) if want_dz else None), N
        colsum = torch.empty(N, dtype=torch.float32, device=dy.device)
        nb = self._lib.tzk_act_bwd_colsum_workspace_bytes(M, N)
        ws = self._workspace("colsum", nb, dy.device)
        check(self._lib.tzk_act_bwd_colsum(_ptr(dy), ld_dy, _ptr(y), ld_y, M, N, int(relu), _ptr(dz), ld_dz,
                                           _ptr(colsum), _ptr(ws), ws.numel(), _stream()), "tzk_act_bwd_colsum")
        self.launches += 2
        return dz, colsum
    # ------------------------------------------------------------------ narrow layers + BCE head
    def small_linear_fwd(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor],
                         relu: bool) -> torch.Tensor:
        x, ld_x = _rows2d(x, "x")
        _need(w, torch.float32, "w")
        M, K = x.shape
        N = w.shape[0]
        if w.shape[1] != K:
            raise TzkError(f"small_linear_fwd: x has {K} columns, w expects {w.shape[1]}")
        y = torch.empty((M, N), dtype=torch.float32, device=x.device)
        if M:
            check(self._lib.tzk_small_linear_fwd(_ptr(x), ld_x, _ptr(w), _ptr(bias), M, K, N, int(relu), _ptr(y), N,
                                                 _stream()), "tzk_small_linear_fwd")
            self.launches += 1
        return y

    def small_linear_bwd(self, x: torch.Tensor, w: torch.Tensor, y: Optional[torch.Tensor], dy: torch.Tensor,
                         relu: bool, want_dx: bool, want_db: bool):
        """-> (dx | None, dw [N,K], db [N] | None)."""
        x, ld_x = _rows2d(x, "x")
        dy, ld_dy = _rows2d(dy, "dy")
        _need(w, torch.float32, "w")
        M, K = x.shape
        N = w.shape[0]
        ld_y = 0
        if relu:
            y, ld_y = _rows2d(y, "y")
        dx = torch.empty((M, K), dtype=torch.float32, device=x.device) if want_dx else None
        dw = torch.empty((N, K), dtype=torch.float32, device=x.device)
        db = torch.empty(N, dtype=torch.float32, device=x.device) if want_db else None
        nb = self._lib.tzk_small_linear_bwd_workspace_bytes(M, K, N)
        ws = self._workspace(("slb", K, N), nb, x.device)
        check(self._lib.tzk_small_linear_bwd(_ptr(x), ld_x, _ptr(w), _ptr(y) if relu else None, ld_y, _ptr(dy), ld_dy,
                                             M, K, N, int(relu), _ptr(dx), K, _ptr(dw), _ptr(db), _ptr(ws),
                                             ws.numel(), _stream()), "tzk_small_linear_bwd")
        # tile kernel + reduction, or (tzk_tower_bwd2.cuh) dx rows kernel + dW kernel + reduction
        self.launches += (2 + int(want_dx)) if _small_linear_rows_path(K, N) else 2
        return dx, dw, db

    def bce_logits_fwd_bwd(self, logits: torch.Tensor, labels: torch.Tensor, want_grad: bool = True):
        """-> (loss [scalar tensor], dloss/dlogits [M] | None); mean reduction."""
        _need(logits, torch.float32, "logits")
        _need(labels, torch.float32, "labels")
        M = logits.numel()
        if labels.numel() != M:
            raise TzkError("bce_logits: logits and labels differ in size")
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        dz = torch.empty(M, dtype=torch.float32, device=logits.device) if want_grad else None
        nb = self._lib.tzk_bce_logits_workspace_bytes(M)
        ws = self._workspace("bce", nb, logits.device)
        check(self._lib.tzk_bce_logits_fwd_bwd(_ptr(logits), _ptr(labels), M, _ptr(loss), _ptr(dz), _ptr(ws),
                                               ws.numel(), _stream()), "tzk_bce_logits_fwd_bwd")
        self.launches += 2
        return loss, dz

    def tower_tail_bce(self, y1: torch.Tensor, w1: torch.Tensor, b1: Optional[torch.Tensor], w2: torch.Tensor,
                       b2: Optional[torch.Tensor], labels: torch.Tensor, relu_dz: bool = False):
        """Last Perceptron (K -> N, ReLU) + Linear(N, 1) + mean BCE, forward and backward in one pass
        (csrc/tzk_tower_tail.cuh).  -> (loss [scalar], logits [M], dy1 [M, K], dW1 [N, K], db1 [N], dw2 [1, N], db2 [1],
        None).  relu_dz (y1 a ReLU output): dz = dy1 * (y1 > 0) in place of dy1, and its column sums [K] last."""
        y1, ld = _rows2d(y1, "y1")
        _need(w1, torch.float32, "w1")
        _need(w2, torch.float32, "w2")
        _need(labels, torch.float32, "labels")
        M, K = y1.shape
        N = w1.shape[0]
        if w1.shape != (N, K) or w2.numel() != N or labels.numel() != M:
            raise TzkError("tower_tail_bce: shapes do not chain")
        dev = y1.device
        logits = torch.empty(M, dtype=torch.float32, device=dev)
        dy1 = torch.empty((M, K), dtype=torch.float32, device=dev)
        out = torch.empty(N * K + 2 * N + 2, dtype=torch.float32, device=dev)
        colsum = torch.empty(K, dtype=torch.float32, device=dev) if relu_dz else None
        nb = self._lib.tzk_tower_tail_bce_workspace_bytes(M, K, N)
        ws = self._workspace("tail", nb, dev)
        check(self._lib.tzk_tower_tail_bce(_ptr(y1), ld, _ptr(w1), _ptr(b1), _ptr(w2), _ptr(b2), _ptr(labels), M, K, N,
                                           _ptr(logits), _ptr(dy1), K, _ptr(colsum), _ptr(out), _ptr(ws), ws.numel(),
                                           _stream()), "tzk_tower_tail_bce")
        self.launches += 3 if relu_dz else 2
        o = N * K
        return (out[o + 2 * N + 1], logits, dy1, out[:o].view(N, K), out[o:o + N], out[o + N:o + 2 * N].view(1, N),
                out[o + 2 * N:o + 2 * N + 1], colsum)

    def binned_auc_update(self, preds: torch.Tensor, labels: torch.Tensor, thresholds: torch.Tensor,
                          counts: torch.Tensor, invalid: torch.Tensor) -> None:
        """counts [T + 1, 2] int64 += the histogram of bin(p) = #{k : p >= thresholds[k]} by label; invalid [1] int64 +=
        the samples with a label outside {0, 1} or a prediction NaN / outside [0, 1] (csrc/tzk_metrics.cuh).
        preds fp32 or bf16, labels fp32 or int64, n of each; thresholds fp32 [T], nondecreasing (not checked here)."""
        if preds.dtype not in (torch.float32, torch.bfloat16):
            raise TzkError(f"binned_auc_update: predictions must be float32 or bfloat16, got {preds.dtype}")
        if labels.dtype not in (torch.float32, torch.int64):
            raise TzkError(f"binned_auc_update: labels must be float32 or int64, got {labels.dtype}")
        _need(preds, preds.dtype, "preds")
        _need(labels, labels.dtype, "labels")
        _need(thresholds, torch.float32, "thresholds")
        _need(counts, torch.int64, "counts")
        _need(invalid, torch.int64, "invalid")
        n, T = preds.numel(), thresholds.numel()
        if labels.numel() != n:
            raise TzkError(f"binned_auc_update: {n} predictions but {labels.numel()} labels")
        if T < 1 or counts.numel() != 2 * (T + 1) or invalid.numel() != 1:
            raise TzkError("binned_auc_update: counts must be [T + 1, 2] and invalid [1] for T >= 1 thresholds")
        check(self._lib.tzk_binned_auc_update(_ptr(preds), int(preds.dtype == torch.bfloat16), _ptr(labels),
                                              int(labels.dtype == torch.int64), n, _ptr(thresholds), T, _ptr(counts),
                                              _ptr(invalid), _stream()), "tzk_binned_auc_update")
        self.launches += int(n > 0)

    # ------------------------------------------------------------------ batch sums of the dense models' kernels
    # (csrc/tzk_batch_sum.cuh).  Every CTA of a backward launch writes its share of the weight, gamma, beta and bias
    # gradients as one row of `partials`, and the rows are added in CTA order: the grid fixes the order of the sums, so
    # it depends only on the work, the shapes and the device.
    def _grid(self, work: int, per_sm: int, slices: int = 1) -> int:
        """CTAs along the work of a launch with `slices` CTAs in grid.y: min(work, ceil(per_sm x SMs / slices))."""
        sms = getattr(self, "_sms", None)
        if sms is None:
            sms = self._sms = max(1, int(self._lib.tzk_sm_count()))
        return max(1, min(int(work), -(-per_sm * sms // slices)))

    def _batch_sums(self, key: str, grid: int, shapes, device):
        """(partials, dparams, views): the cached workspace `key` for `grid` rows of partials, dparams, and dparams cut
        into views of `shapes` in the order the kernel writes them."""
        sizes = [math.prod(s) for s in shapes]
        partials = self._workspace(key, grid * sum(sizes) * 4, device)
        dparams = torch.empty(sum(sizes), dtype=torch.float32, device=device)
        return partials, dparams, [v.view(s) for v, s in zip(dparams.split(sizes), shapes)]

    # ------------------------------------------------------------------ WuKong layer (csrc/tzk_wukong.cuh)
    def wukong_mix_fwd(self, x, w_fmb, gamma, beta, w_lcb, w_res, f: int):
        """x [B, n, d] -> (ln_f [B, n k], stats [B, 2], base [B, f + l, d]); w_res None: identity residual."""
        for t, nm in ((x, "x"), (w_fmb, "w_fmb"), (gamma, "gamma"), (beta, "beta"), (w_lcb, "w_lcb")):
            _need(t, torch.float32, nm)
        if w_res is not None:
            _need(w_res, torch.float32, "w_res")
        B, n, d = x.shape
        k, l = w_fmb.shape[1], w_lcb.shape[1]
        m = f + l
        ln_f = torch.empty((B, n * k), dtype=torch.float32, device=x.device)
        stats = torch.empty((B, 2), dtype=torch.float32, device=x.device)
        base = torch.empty((B, m, d), dtype=torch.float32, device=x.device)
        check(self._lib.tzk_wukong_mix_fwd(_ptr(x), _ptr(w_fmb), _ptr(gamma), _ptr(beta), _ptr(w_lcb), _ptr(w_res), B,
                                           n, d, k, f, l, self._grid(B, 8), _ptr(ln_f), _ptr(stats), _ptr(base),
                                           _stream()), "tzk_wukong_mix_fwd")
        self.launches += int(B > 0)
        return ln_f, stats, base

    def wukong_mix_bwd(self, x, w_fmb, gamma, w_lcb, w_res, f: int, stats, d_ln_f, d_base):
        """-> (dx, dw_fmb, dgamma, dbeta, dw_lcb, dw_res or None)."""
        for t, nm in ((x, "x"), (w_fmb, "w_fmb"), (gamma, "gamma"), (w_lcb, "w_lcb"), (stats, "stats"),
                      (d_ln_f, "d_ln_f"), (d_base, "d_base")):
            _need(t, torch.float32, nm)
        if w_res is not None:
            _need(w_res, torch.float32, "w_res")
        B, n, d = x.shape
        k, l = w_fmb.shape[1], w_lcb.shape[1]
        m = f + l
        grid = self._grid(B, 4)       # mix_bwd_kernel: 4 resident CTAs per SM (launch bounds)
        dx = torch.empty_like(x)
        partials, dparams, (dw_fmb, dw_lcb, dw_res, dgamma, dbeta) = self._batch_sums(
            "wukong_mix_bwd", grid, [(n, k), (n, l), (n, m if w_res is not None else 0), (n * k,), (n * k,)], x.device)
        check(self._lib.tzk_wukong_mix_bwd(_ptr(x), _ptr(w_fmb), _ptr(gamma), _ptr(w_lcb), _ptr(w_res), _ptr(stats),
                                           _ptr(d_ln_f), _ptr(d_base), B, n, d, k, f, l, grid, _ptr(dx),
                                           _ptr(partials), _ptr(dparams), _stream()), "tzk_wukong_mix_bwd")
        self.launches += 1 + int(B > 0)
        return dx, dw_fmb, dgamma, dbeta, dw_lcb, (dw_res if w_res is not None else None)

    def wukong_out_fwd(self, fmb_out, base, gamma, beta, f: int):
        """fmb_out [B, f d], base [B, m, d] -> (y [B, m, d], stats [B, m, 2])."""
        for t, nm in ((fmb_out, "fmb_out"), (base, "base"), (gamma, "gamma"), (beta, "beta")):
            _need(t, torch.float32, nm)
        B, m, d = base.shape
        y = torch.empty_like(base)
        stats = torch.empty((B, m, 2), dtype=torch.float32, device=base.device)
        check(self._lib.tzk_wukong_out_fwd(_ptr(fmb_out), _ptr(base), _ptr(gamma), _ptr(beta), B, d, f, m - f,
                                           self._grid(-(-B * m // 128), 8), _ptr(y), _ptr(stats), _stream()),
              "tzk_wukong_out_fwd")
        self.launches += int(B > 0)
        return y, stats

    def wukong_out_bwd(self, fmb_out, base, gamma, f: int, stats, dy):
        """-> (d_fmb_out [B, f d], d_base [B, m, d], dgamma [d], dbeta [d])."""
        for t, nm in ((fmb_out, "fmb_out"), (base, "base"), (gamma, "gamma"), (stats, "stats"), (dy, "dy")):
            _need(t, torch.float32, nm)
        B, m, d = base.shape
        grid = self._grid(-(-B * m // 128), 4)
        d_fmb = torch.empty_like(fmb_out)
        d_base = torch.empty_like(base)
        partials, dparams, (dgamma, dbeta) = self._batch_sums("wukong_out_bwd", grid, [(d,), (d,)], base.device)
        check(self._lib.tzk_wukong_out_bwd(_ptr(fmb_out), _ptr(base), _ptr(gamma), _ptr(stats), _ptr(dy), B, d, f,
                                           m - f, grid, _ptr(d_fmb), _ptr(d_base), _ptr(partials), _ptr(dparams),
                                           _stream()), "tzk_wukong_out_bwd")
        self.launches += 1 + int(B > 0)
        return d_fmb, d_base, dgamma, dbeta

    # ------------------------------------------------------------------ MaskNet (csrc/tzk_masknet.cuh)
    # CTAs per SM of each launch (ptxas register counts at 128 threads: mask_fwd 45, mask_bwd 70, ffn_fwd 78,
    # ffn_bwd 96); the FFN launches have one grid.y slice per mask block.

    def masknet_mask_fwd(self, e, m, b2, gamma, beta, E: int, nb: int):
        """e [B, Ep] (first E columns live), m [B, nb Ep] -> (v [B, nb Ep], stats [B, 2]); Ep = pad4(E)."""
        for t, nm in ((e, "e"), (m, "m"), (b2, "b2"), (gamma, "gamma"), (beta, "beta")):
            _need(t, torch.float32, nm)
        B = e.shape[0]
        v = torch.empty_like(m)
        stats = torch.empty((B, 2), dtype=torch.float32, device=e.device)
        check(self._lib.tzk_masknet_mask_fwd(_ptr(e), e.shape[1], _ptr(m), _ptr(b2), _ptr(gamma), _ptr(beta), B, E, nb,
                                             self._grid(B, 8), _ptr(v), _ptr(stats), _stream()),
              "tzk_masknet_mask_fwd")
        self.launches += int(B > 0)
        return v, stats

    def masknet_mask_bwd(self, e, m, b2, gamma, beta, stats, dv, E: int, nb: int):
        """-> (dm [B, nb Ep], de [B, Ep], db2 [nb E], dgamma [E], dbeta [E])."""
        for t, nm in ((e, "e"), (m, "m"), (b2, "b2"), (gamma, "gamma"), (beta, "beta"), (stats, "stats"),
                      (dv, "dv")):
            _need(t, torch.float32, nm)
        B = e.shape[0]
        grid = self._grid(B, 6)
        dm = torch.empty_like(m)
        de = torch.empty_like(e)
        partials, dparams, (db2, dgamma, dbeta) = self._batch_sums("masknet_mask_bwd", grid, [(nb * E,), (E,), (E,)],
                                                                   e.device)
        check(self._lib.tzk_masknet_mask_bwd(_ptr(e), e.shape[1], _ptr(m), _ptr(b2), _ptr(gamma), _ptr(beta),
                                             _ptr(stats), _ptr(dv), B, E, nb, grid, _ptr(dm), _ptr(de),
                                             _ptr(partials), _ptr(dparams), _stream()), "tzk_masknet_mask_bwd")
        self.launches += 1 + int(B > 0)
        return dm, de, db2, dgamma, dbeta

    def masknet_ffn_fwd(self, z, b3, gamma, beta, nb: int):
        """z [B, nb H] -> (y [B, nb H] = ReLU(LN_H(z_i + b3_i)) per block, stats [B, nb, 2])."""
        for t, nm in ((z, "z"), (b3, "b3"), (gamma, "gamma"), (beta, "beta")):
            _need(t, torch.float32, nm)
        B, H = z.shape[0], z.shape[1] // nb
        y = torch.empty_like(z)
        stats = torch.empty((B, nb, 2), dtype=torch.float32, device=z.device)
        check(self._lib.tzk_masknet_ffn_fwd(_ptr(z), _ptr(b3), _ptr(gamma), _ptr(beta), B, H, nb,
                                            self._grid(B, 6, nb), _ptr(y), _ptr(stats), _stream()),
              "tzk_masknet_ffn_fwd")
        self.launches += int(B > 0)
        return y, stats

    def masknet_ffn_bwd(self, z, b3, gamma, beta, stats, dy, nb: int):
        """-> (dz [B, nb H], dgamma [nb, H], dbeta [nb, H], db3 [nb, H])."""
        for t, nm in ((z, "z"), (b3, "b3"), (gamma, "gamma"), (beta, "beta"), (stats, "stats"), (dy, "dy")):
            _need(t, torch.float32, nm)
        B, H = z.shape[0], z.shape[1] // nb
        grid = self._grid(B, 5, nb)
        dz = torch.empty_like(z)
        partials, dparams, (g3,) = self._batch_sums("masknet_ffn_bwd", grid, [(nb, 3, H)], z.device)
        check(self._lib.tzk_masknet_ffn_bwd(_ptr(z), _ptr(b3), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(dy), B, H,
                                            nb, grid, _ptr(dz), _ptr(partials), _ptr(dparams), _stream()),
              "tzk_masknet_ffn_bwd")
        self.launches += 1 + int(B > 0)
        return dz, g3[:, 0], g3[:, 1], g3[:, 2]

    # ------------------------------------------------------------------ PLE gates (csrc/tzk_ple.cuh)
    # Resident CTAs per SM: ptxas register counts at 256 threads (gate_fwd 58 -> 4, gate_bwd 79 -> 3), fewer when the
    # layer's shared memory (tzk_ple_gate_smem_bytes) allows fewer.  The grid fixes the order of the batch sums and
    # depends only on the batch size, the layer's shapes and the device.
    def _ple_args(self, inputs, gate_input, weights, biases, experts, gate_experts, d_inputs=None):
        from ._lib import TzkPleGateArgs

        a = TzkPleGateArgs()
        a.B, a.H = experts[0].shape[0], experts[0].shape[1]
        a.n_experts, a.n_inputs, a.n_gates = len(experts), len(inputs), len(gate_input)
        for i, x in enumerate(inputs):
            _need(x, torch.float32, f"inputs[{i}]")
            a.in_dim[i], a.inputs[i] = x.shape[1], x.data_ptr()
            if d_inputs is not None:
                a.d_inputs[i] = d_inputs[i].data_ptr()
        for j, e in enumerate(experts):
            _need(e, torch.float32, f"experts[{j}]")
            if tuple(e.shape) != (a.B, a.H):
                raise TzkError("ple gates: every expert output must have the same [B, H] shape")
            a.experts[j] = e.data_ptr()
        for g, (w, b) in enumerate(zip(weights, biases)):
            _need(w, torch.float32, f"weight[{g}]")
            _need(b, torch.float32, f"bias[{g}]")
            a.gate_input[g], a.gate_num_experts[g] = gate_input[g], len(gate_experts[g])
            for e, x in enumerate(gate_experts[g]):
                a.gate_experts[g][e] = x
            a.weight[g], a.bias[g] = w.data_ptr(), b.data_ptr()
        return a

    def _ple_grid(self, a, B: int, rows_per_cta: int, per_sm_regs: int, backward: int) -> int:
        smem = int(self._lib.tzk_ple_gate_smem_bytes(ctypes.byref(a), backward))
        if smem == 0:
            raise TzkError("ple gates: layer outside the kernels' cover (Fn.ple_gate_usable)")
        per_sm = max(1, min(per_sm_regs, (227 * 1024) // (smem + 1024)))
        return self._grid(-(-int(B) // rows_per_cta), per_sm)

    def ple_gate_fwd(self, inputs, gate_input, weights, biases, experts, gate_experts):
        """One extraction layer's gates -> (y [n_gates, B, H], p [B, sum E_g] the softmax of every gate)."""
        a = self._ple_args(inputs, gate_input, weights, biases, experts, gate_experts)
        B, H, G = a.B, a.H, a.n_gates
        dev = experts[0].device
        y = torch.empty((G, B, H), dtype=torch.float32, device=dev)
        p = torch.empty((B, sum(len(e) for e in gate_experts)), dtype=torch.float32, device=dev)
        grid = self._ple_grid(a, B, 8, 4, 0)
        check(self._lib.tzk_ple_gate_fwd(ctypes.byref(a), grid, _ptr(y), _ptr(p), _stream()), "tzk_ple_gate_fwd")
        self.launches += int(B > 0)
        return y, p

    def ple_gate_bwd(self, inputs, gate_input, weights, biases, experts, gate_experts, p, dy):
        """dy [n_gates, B, H] -> (d_inputs [B, K_i] per input, d_experts [n_experts, B, H], dW_g per gate, db_g per
        gate)."""
        _need(p, torch.float32, "p")
        _need(dy, torch.float32, "dy")
        d_inputs = [torch.empty_like(x) for x in inputs]
        a = self._ple_args(inputs, gate_input, weights, biases, experts, gate_experts, d_inputs)
        B, H = a.B, a.H
        dev = experts[0].device
        grid = self._ple_grid(a, B, 16, 3, 1)
        d_experts = torch.empty((len(experts), B, H), dtype=torch.float32, device=dev)
        partials, dparams, views = self._batch_sums(
            "ple_gate_bwd", grid, [tuple(w.shape) for w in weights] + [(len(e),) for e in gate_experts], dev)
        check(self._lib.tzk_ple_gate_bwd(ctypes.byref(a), _ptr(p), _ptr(dy), grid, _ptr(d_experts), _ptr(partials),
                                         _ptr(dparams), _stream()), "tzk_ple_gate_bwd")
        self.launches += 1 + int(B > 0)
        return d_inputs, d_experts, views[:len(weights)], views[len(weights):]

    # ------------------------------------------------------------------ PEPNet gate product (csrc/tzk_pepnet.cuh)
    # Resident CTAs per SM: ptxas register counts at 256 threads (gate_fwd 35 -> 6, gate_bwd 72 -> 3).  The grid fixes
    # the order of the batch sums and depends only on the batch size, the segments' widths and the device.
    def _pepnet_args(self, segs, dys=None, dxs=None, dzs=None):
        """segs: [(x, bx, z, bz, y, relu, gamma)], x / z / y [B, N] views with contiguous rows, bx None or [N]."""
        from ._lib import PEPNET_MAX_SEGS, PEPNET_IDENTITY, PEPNET_RELU, TzkPepnetGateArgs

        if not 1 <= len(segs) <= PEPNET_MAX_SEGS:
            raise TzkError(f"pepnet gates: 1..{PEPNET_MAX_SEGS} segments, got {len(segs)}")
        a = TzkPepnetGateArgs()
        a.B, a.n_segs = segs[0][0].shape[0], len(segs)
        for s, (x, bx, z, bz, y, relu, gamma) in enumerate(segs):
            x, ldx = _rows2d(x, f"x[{s}]")
            z, ldz = _rows2d(z, f"z[{s}]")
            g = a.seg[s]
            g.x, g.z, g.bz = x.data_ptr(), z.data_ptr(), _need(bz, torch.float32, f"bz[{s}]").data_ptr()
            g.bx = None if bx is None else _need(bx, torch.float32, f"bx[{s}]").data_ptr()
            g.ldx, g.ldz, g.N = ldx, ldz, x.shape[1]
            g.act, g.gamma = (PEPNET_RELU if relu else PEPNET_IDENTITY), float(gamma)
            if y is not None:
                y, g.ldy = _rows2d(y, f"y[{s}]")
                g.y = y.data_ptr()
            if dys is not None:
                dy, g.ldy = _rows2d(dys[s], f"dy[{s}]")
                _, ld_dx = _rows2d(dxs[s], f"dx[{s}]")
                _, ld_dz = _rows2d(dzs[s], f"dz[{s}]")
                if (ld_dx, ld_dz) != (ldx, ldz):
                    raise TzkError("pepnet_gate_bwd: dx / dz must have the row pitches of x / z")
                g.dy, g.dx, g.dz = dy.data_ptr(), dxs[s].data_ptr(), dzs[s].data_ptr()
            if tuple(z.shape) != tuple(x.shape) or x.shape[0] != a.B:
                raise TzkError("pepnet gates: x and z of a segment must have one [B, N] shape")
        return a

    def _pepnet_grid(self, a, per_sm: int) -> int:
        rows = min(256 // (a.seg[s].N // 4) for s in range(a.n_segs))
        return self._grid(-(-int(a.B) // rows), per_sm, a.n_segs)

    def pepnet_gate_fwd(self, segs):
        """y = act(x + bx) * gamma sigmoid(z + bz) into every segment's y (written in place)."""
        a = self._pepnet_args(segs)
        check(self._lib.tzk_pepnet_gate_fwd(ctypes.byref(a), self._pepnet_grid(a, 6), _stream()),
              "tzk_pepnet_gate_fwd")
        self.launches += int(a.B > 0)

    def pepnet_gate_bwd(self, segs, dys, dxs, dzs):
        """dys -> dxs, dzs (written in place), returns [(dbx, dbz)] per segment."""
        a = self._pepnet_args(segs, dys, dxs, dzs)
        dev = segs[0][0].device
        grid = self._pepnet_grid(a, 3)
        partials, dparams, views = self._batch_sums("pepnet_gate_bwd", grid,
                                                    [(s[0].shape[1],) for s in segs for _ in range(2)], dev)
        check(self._lib.tzk_pepnet_gate_bwd(ctypes.byref(a), grid, _ptr(partials), _ptr(dparams), _stream()),
              "tzk_pepnet_gate_bwd")
        self.launches += 1 + int(a.B > 0)
        return list(zip(views[0::2], views[1::2]))

    # ------------------------------------------------------------------ JRC loss (csrc/tzk_jrc.cuh)
    def jrc_loss(self, logits: torch.Tensor, labels: torch.Tensor, session_ids: torch.Tensor,
                 weights: Optional[torch.Tensor], alpha: float, key_bits: int = 64):
        """logits [B, 2] fp32 (contiguous rows), labels [B] fp32, session_ids [B] int64 in [0, 2^key_bits), weights [B]
        fp32 or None (mean reduction) -> (loss [scalar], d loss / d logits [B, 2])."""
        logits, ld = _rows2d(logits, "logits")
        _need(labels, torch.float32, "labels")
        _need(session_ids, torch.int64, "session_ids")
        if weights is not None:
            _need(weights, torch.float32, "weights")
        B = logits.shape[0]
        if logits.shape[1] != 2 or labels.numel() != B or session_ids.numel() != B or (
                weights is not None and weights.numel() != B):
            raise TzkError("jrc_loss: need logits [B, 2] and B labels, session ids (and weights)")
        dev = logits.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        dlogits = torch.empty((B, 2), dtype=torch.float32, device=dev)
        ws = self._workspace("jrc", self._lib.tzk_jrc_loss_workspace_bytes(B), dev)
        check(self._lib.tzk_jrc_loss(_ptr(logits), ld, _ptr(labels), _ptr(session_ids), _ptr(weights), B, float(alpha),
                                     int(key_bits), _ptr(loss), _ptr(dlogits), _ptr(ws), ws.numel(), _stream()),
              "tzk_jrc_loss")
        self.launches += 6 if B > 0 else 1            # iota, pass 1-3 and two carries; B = 0: one carry (CUB's sort not counted)
        return loss, dlogits

    # ------------------------------------------------------------------ RocketLaunching head (csrc/tzk_rocket.cuh)
    # Resident CTAs per SM: ptxas register counts at 256 threads (head_fwd 80 -> 3, head_bwd 48 -> 5).  The grid fixes
    # the order of the loss and parameter sums and depends only on the batch size and the device.
    def _rocket_args(self, heads, logits, probs, labels, eps: float, pairs, sim: int, pair_stats, dhs=None,
                     dlights=None):
        from ._lib import ROCKET_MAX_PAIRS, TzkRocketArgs

        if not 1 <= len(heads) <= 2 or len(pairs) > ROCKET_MAX_PAIRS:
            raise TzkError(f"rocket head: 1 or 2 heads and at most {ROCKET_MAX_PAIRS} pairs")
        a = TzkRocketArgs()
        B, C = heads[0][0].shape[0], heads[0][1].shape[0]
        a.B, a.C, a.has_booster, a.n_pairs, a.sim, a.eps = B, C, len(heads) - 1, len(pairs), int(sim), float(eps)
        if labels is not None:
            a.labels = _need(labels, torch.float32, "labels").data_ptr()
            if labels.numel() != B:
                raise TzkError("rocket head: need one label per sample")
        a.pair_stats = _ptr(pair_stats)
        for e, (h, w, b) in enumerate(heads):
            for t, nm in ((h, "h"), (w, "w"), (b, "b"), (logits[e], "logits"), (probs[e], "probs")):
                _need(t, torch.float32, f"head[{e}].{nm}")
            if h.shape[0] != B or tuple(w.shape) != (C, h.shape[1]) or b.numel() != C:
                raise TzkError("rocket head: need h [B, H], w [C, H] and b [C] with one B and one C")
            g = a.head[e]
            g.h, g.w, g.b, g.logits, g.probs, g.H = h.data_ptr(), w.data_ptr(), b.data_ptr(), logits[e].data_ptr(), \
                probs[e].data_ptr(), h.shape[1]
            if dhs is not None:
                g.dh = dhs[e].data_ptr()
        for k, (l, o) in enumerate(pairs):
            _need(l, torch.float32, f"pair[{k}].light")
            _need(o, torch.float32, f"pair[{k}].booster")
            if l.shape != o.shape or l.shape[0] != B:
                raise TzkError("rocket head: the light and booster layers of a pair must have one [B, d] shape")
            p = a.pair[k]
            p.light, p.booster, p.d = l.data_ptr(), o.data_ptr(), l.shape[1]
            if dlights is not None:
                p.dlight = dlights[k].data_ptr()
        return a

    def rocket_head_fwd(self, heads, labels, eps: float, pairs, sim: int):
        """heads [(h [B, H], w [C, H], b [C])]: the light head, then optionally the booster head; labels [B] fp32 class
        indices or None; pairs [(light [B, d], booster [B, d])] -> (logits per head, probs per head, losses
        [3 + n_pairs] or None, pair_stats or None)."""
        dev = heads[0][0].device
        B, C = heads[0][0].shape[0], heads[0][1].shape[0]
        logits = [torch.empty((B, C), dtype=torch.float32, device=dev) for _ in heads]
        probs = [torch.empty((B, C), dtype=torch.float32, device=dev) for _ in heads]
        pair_stats = torch.empty((len(pairs), B, 2), dtype=torch.float32, device=dev) if pairs else None
        losses = partials = None
        grid = self._grid(-(-int(B) // 8), 3)
        if labels is not None:
            losses = torch.empty(3 + len(pairs), dtype=torch.float32, device=dev)
            partials = self._workspace("rocket_fwd", grid * losses.numel() * 4, dev)
        a = self._rocket_args(heads, logits, probs, labels, eps, pairs, sim, pair_stats)
        check(self._lib.tzk_rocket_head_fwd(ctypes.byref(a), grid, _ptr(partials), _ptr(losses), _stream()),
              "tzk_rocket_head_fwd")
        self.launches += int(B > 0) + int(labels is not None)
        return logits, probs, losses, pair_stats

    def rocket_head_bwd(self, heads, logits, probs, labels, eps: float, pairs, sim: int, pair_stats, losses, dlosses):
        """dlosses [3 + n_pairs] (device) -> (dh per head, dlight per pair, [(dW [C, H], db [C])] per head)."""
        _need(losses, torch.float32, "losses")
        _need(dlosses, torch.float32, "dlosses")
        dev = heads[0][0].device
        B, C = heads[0][0].shape[0], heads[0][1].shape[0]
        dhs = [torch.empty_like(h) for h, _, _ in heads]
        dlights = [torch.empty_like(l) for l, _ in pairs]
        a = self._rocket_args(heads, logits, probs, labels, eps, pairs, sim, pair_stats, dhs, dlights)
        grid = self._grid(-(-int(B) // 32), 5)
        shapes = [s for h, _, _ in heads for s in ((C, h.shape[1]), (C,))]
        partials, dparams, views = self._batch_sums("rocket_bwd", grid, shapes, dev)
        check(self._lib.tzk_rocket_head_bwd(ctypes.byref(a), _ptr(dlosses), _ptr(losses), grid, _ptr(partials),
                                            _ptr(dparams), _stream()), "tzk_rocket_head_bwd")
        self.launches += 1 + int(B > 0)
        return dhs, dlights, list(zip(views[0::2], views[1::2]))


    # ------------------------------------------------------------------ TDM multi-window DIN (csrc/tzk_tdm.cuh)
    # Resident CTAs per SM: ptxas register counts (fwd 61 at 256 threads -> 4, bwd 126 at 128 threads -> 4), fewer when
    # the shapes' shared memory (tzk_tdm_smem_bytes) allows fewer.  The backward grid fixes the order of the parameter
    # sums and depends only on the batch size, the shapes and the device.
    def _tdm_args(self, query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu: bool):
        from ._lib import TDM_MAX_LAYERS, TDM_MAX_WINDOWS, TDM_PRELU, TDM_RELU, TzkTdmArgs

        _need(query, torch.float32, "query")
        _need(seq, torch.float32, "seq")
        _need(offsets, torch.int64, "offsets")
        if not 1 <= len(layers) <= TDM_MAX_LAYERS or not 1 <= len(windows) <= TDM_MAX_WINDOWS:
            raise TzkError(f"tdm: 1..{TDM_MAX_LAYERS} attention layers and 1..{TDM_MAX_WINDOWS} windows")
        a = TzkTdmArgs()
        a.B, a.Dq = query.shape
        a.N, a.C = seq.shape
        if offsets.numel() != a.B + 1:
            raise TzkError("tdm: need offsets [B + 1] for query [B, Dq]")
        a.L, a.n_layers, a.act = len(windows), len(layers), TDM_PRELU if prelu else TDM_RELU
        for w, n in enumerate(windows):
            a.windows[w] = int(n)
        a.seq, a.offsets, a.query = seq.data_ptr(), offsets.data_ptr(), query.data_ptr()
        K = 3 * a.C
        for l, (W, b, slope) in enumerate(layers):
            _need(W, torch.float32, f"w[{l}]")
            _need(b, torch.float32, f"b[{l}]")
            if W.dim() != 2 or W.shape[1] != K or b.numel() != W.shape[0]:
                raise TzkError(f"tdm: layer {l} needs w [H, {K}] and b [H]")
            a.hidden[l], a.w[l], a.b[l] = W.shape[0], W.data_ptr(), b.data_ptr()
            if prelu:
                a.slope[l] = _need(slope, torch.float32, f"slope[{l}]").data_ptr()
            K = W.shape[0]
        for t, nm in ((lin_w, "lin_w"), (lin_b, "lin_b"), (act_w, "act_w")):
            _need(t, torch.float32, nm)
        if lin_w.numel() != K or lin_b.numel() != 1 or act_w.numel() != 1:
            raise TzkError("tdm: need lin_w [1, H_last], lin_b [1] and act_w [1]")
        a.lin_w, a.lin_b, a.act_w = lin_w.data_ptr(), lin_b.data_ptr(), act_w.data_ptr()
        return a

    def _tdm_grid(self, a, B: int, backward: int) -> int:
        smem = int(self._lib.tzk_tdm_smem_bytes(ctypes.byref(a), backward))
        if smem == 0:
            raise TzkError("tdm: shapes outside the kernels' cover (Fn.multiwindow_din_usable)")
        per_sm = max(1, min(4, (227 * 1024) // (smem + 1024)))
        return self._grid(-(-int(B) // 8) if not backward else int(B), per_sm)

    def tdm_fwd(self, query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu: bool):
        """query [B, Dq], seq [N, C] jagged rows, offsets [B + 1] int64, layers [(w [H, K], b [H], slope [1] or
        None)], lin_w [1, H_last], lin_b [1], act_w [1] -> (out [B, (L + 1) C], z [N])."""
        a = self._tdm_args(query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu)
        out = torch.empty((a.B, (a.L + 1) * a.C), dtype=torch.float32, device=seq.device)
        z = torch.empty(a.N, dtype=torch.float32, device=seq.device)
        a.out, a.z = out.data_ptr(), z.data_ptr()
        check(self._lib.tzk_tdm_fwd(ctypes.byref(a), self._tdm_grid(a, a.B, 0), _stream()), "tzk_tdm_fwd")
        self.launches += int(a.B > 0)
        return out, z

    def tdm_bwd(self, query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu: bool, z, d_out):
        """-> (d_query [B, Dq], d_seq [N, C], [(dw, db, dslope or None)] per layer, d lin_w, d lin_b, d act_w)."""
        _need(z, torch.float32, "z")
        _need(d_out, torch.float32, "d_out")
        a = self._tdm_args(query, seq, offsets, layers, lin_w, lin_b, act_w, windows, prelu)
        if z.numel() != a.N or tuple(d_out.shape) != (a.B, (a.L + 1) * a.C):
            raise TzkError("tdm_bwd: need z [N] and d_out [B, (L + 1) C]")
        d_query, d_seq = torch.empty_like(query), torch.empty_like(seq)
        a.z, a.d_out, a.d_seq, a.d_query = z.data_ptr(), d_out.data_ptr(), d_seq.data_ptr(), d_query.data_ptr()
        grid = self._tdm_grid(a, a.B, 1)
        shapes = []
        for W, _, _ in layers:
            shapes += [tuple(W.shape), (W.shape[0],)] + ([(1,)] if prelu else [])
        shapes += [tuple(lin_w.shape), (1,), (1,)]
        partials, dparams, views = self._batch_sums("tdm_bwd", grid, shapes, seq.device)
        check(self._lib.tzk_tdm_bwd(ctypes.byref(a), grid, _ptr(partials), _ptr(dparams), _stream()), "tzk_tdm_bwd")
        self.launches += 1 + int(a.B > 0)
        per, grads, o = 3 if prelu else 2, [], 0
        for _ in layers:
            grads.append((views[o], views[o + 1], views[o + 2] if prelu else None))
            o += per
        return d_query, d_seq, grads, views[o], views[o + 1], views[o + 2]

    # ------------------------------------------------------------------ DCN-v2 cross network (csrc/tzk_dcn_v2.cuh)
    # fwd and bwd_data run CTAs of up to 4 warps over 64-row groups: resident CTAs per SM from the shapes' shared
    # memory (tzk_dcn_v2_smem_bytes) and the ptxas register counts (at most 168 registers at 128 threads -> 3).
    # bwd_weight runs (32-column block) x (batch chunk) CTAs of 4 warps (at most 222 registers -> 2 per SM); the chunk
    # count fixes the order of the parameter sums and depends only on the batch size, the shapes and the device.
    def _dcn_v2_args(self, x0, wu, wv, bias):
        from ._lib import TzkDcnV2Args

        _need(x0, torch.float32, "x0")
        for t, nm in ((wu, "wu"), (wv, "wv"), (bias, "bias")):
            _need(t, torch.float32, nm)
        a = TzkDcnV2Args()
        a.B, a.D = x0.shape
        a.L, a.r = wu.shape[0], wu.shape[1]
        if tuple(wu.shape) != (a.L, a.r, a.D) or tuple(wv.shape) != (a.L, a.D, a.r) or tuple(bias.shape) != (a.L, a.D):
            raise TzkError("dcn_v2: need x0 [B, D], wu [L, r, D], wv [L, D, r] and bias [L, D]")
        a.x0, a.wu, a.wv, a.bias = x0.data_ptr(), wu.data_ptr(), wv.data_ptr(), bias.data_ptr()
        r8, d8 = -(-a.r // 8) * 8, -(-a.D // 8) * 8
        work = self._workspace("dcn_v2_work", 8 * a.L * r8 * d8 * 4, x0.device)
        a.work = work.data_ptr()
        return a

    def _dcn_v2_smem(self, a, pass_: int) -> int:
        smem = int(self._lib.tzk_dcn_v2_smem_bytes(ctypes.byref(a), pass_))
        if smem == 0:
            raise TzkError("dcn_v2: shapes outside the kernels' cover (Fn.cross_v2_usable)")
        return smem

    def _dcn_v2_tile_grid(self, a, pass_: int) -> int:
        per_sm = max(1, min(3, (227 * 1024) // (self._dcn_v2_smem(a, pass_) + 1024)))
        return self._grid(-(-int(a.B) // 64), per_sm)

    def dcn_v2_fwd(self, x0, wu, wv, bias):
        """x0 [B, D], wu [L, r, D], wv [L, D, r], bias [L, D] -> (y [B, D], v [B, L r])."""
        a = self._dcn_v2_args(x0, wu, wv, bias)
        y = torch.empty_like(x0)
        v = torch.empty((a.B, a.L * a.r), dtype=torch.float32, device=x0.device)
        a.y, a.v = y.data_ptr(), v.data_ptr()
        check(self._lib.tzk_dcn_v2_fwd(ctypes.byref(a), self._dcn_v2_tile_grid(a, 0), _stream()), "tzk_dcn_v2_fwd")
        self.launches += 2 * int(a.B > 0)
        return y, v

    def dcn_v2_bwd(self, x0, wu, wv, bias, v, dy):
        """-> (dx0 [B, D], d wu [L, r, D], d wv [L, D, r], d bias [L, D]) from the saved v and dy = d y."""
        _need(v, torch.float32, "v")
        _need(dy, torch.float32, "dy")
        a = self._dcn_v2_args(x0, wu, wv, bias)
        if tuple(v.shape) != (a.B, a.L * a.r) or tuple(dy.shape) != (a.B, a.D):
            raise TzkError("dcn_v2_bwd: need v [B, L r] and dy [B, D]")
        dx0 = torch.empty_like(x0)
        dv = torch.empty_like(v)
        a.v, a.dy, a.dx0, a.dv = v.data_ptr(), dy.data_ptr(), dx0.data_ptr(), dv.data_ptr()
        check(self._lib.tzk_dcn_v2_bwd_data(ctypes.byref(a), self._dcn_v2_tile_grid(a, 1), _stream()),
              "tzk_dcn_v2_bwd_data")
        blocks = -(-a.D // 32)
        per_sm = max(1, min(2, (227 * 1024) // (self._dcn_v2_smem(a, 2) + 1024)))
        chunks = self._grid(-(-int(a.B) // 64), per_sm, blocks)
        shapes = [tuple(wu.shape), tuple(wv.shape), tuple(bias.shape)]
        partials, dparams, views = self._batch_sums("dcn_v2_bwd", chunks, shapes, x0.device)
        check(self._lib.tzk_dcn_v2_bwd_weight(ctypes.byref(a), chunks, _ptr(partials), _ptr(dparams), _stream()),
              "tzk_dcn_v2_bwd_weight")
        self.launches += 1 + 5 * int(a.B > 0)
        return dx0, views[0], views[1], views[2]

    # ------------------------------------------------------------------ sequence encoders (csrc/tzk_seq_attn.cuh)
    # The attention core runs one CTA of 256 threads per (sample, head) item at a time, grid-stride; resident CTAs per
    # SM from the ptxas register counts (fwd 100 -> 2, bwd up to 168 -> 1) and the shared memory of hd.  Every item
    # writes only its own outputs, so the grid changes no bits.
    def _seq_attn_args(self, q, k, v, offsets, H: int, max_len: int):
        from ._lib import TzkSeqAttnArgs

        for t, nm in ((q, "q"), (k, "k"), (v, "v")):
            _need(t, torch.float32, nm)
        _need(offsets, torch.int64, "offsets")
        a = TzkSeqAttnArgs()
        a.N, E = q.shape
        a.B, a.H, a.max_len = offsets.numel() - 1, int(H), int(max_len)
        if a.B < 0 or H < 1 or E % H != 0 or q.dim() != 2 or tuple(k.shape) != (a.N, E) or tuple(v.shape) != (a.N, E):
            raise TzkError("self_attn_pool: need q, k, v [N, H hd] and offsets [B + 1]")
        a.hd = E // H
        a.ldq = a.ldk = a.ldv = E
        a.offsets, a.q, a.k, a.v = offsets.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr()
        return a

    def _seq_attn_grid(self, a, backward: bool) -> int:
        smem = int(self._lib.tzk_seq_attn_smem_bytes(ctypes.byref(a)))
        if smem == 0:
            raise TzkError("self_attn_pool: shapes outside the kernels' cover (Fn.self_attn_pool_usable)")
        per_sm = max(1, min(1 if backward else 2, (227 * 1024) // (smem + 1024)))
        return self._grid(int(a.B) * int(a.H), per_sm)

    def self_attn_pool_fwd(self, q, k, v, offsets, H: int, max_len: int):
        """q, k, v [N, E], offsets [B + 1] int64 -> (pooled [B, E], lse [N, H])."""
        a = self._seq_attn_args(q, k, v, offsets, H, max_len)
        pooled = torch.empty((a.B, a.H * a.hd), dtype=torch.float32, device=q.device)
        lse = torch.empty((a.N, a.H), dtype=torch.float32, device=q.device)
        a.pooled, a.lse = pooled.data_ptr(), lse.data_ptr()
        check(self._lib.tzk_self_attn_pool_fwd(ctypes.byref(a), self._seq_attn_grid(a, False), _stream()),
              "tzk_self_attn_pool_fwd")
        self.launches += int(a.B > 0)
        return pooled, lse

    def self_attn_pool_bwd(self, q, k, v, offsets, H: int, max_len: int, lse, d_pooled):
        """-> (dq, dk, dv [N, E]) from the saved lse [N, H] and d_pooled [B, E]."""
        _need(lse, torch.float32, "lse")
        _need(d_pooled, torch.float32, "d_pooled")
        a = self._seq_attn_args(q, k, v, offsets, H, max_len)
        E = a.H * a.hd
        if tuple(lse.shape) != (a.N, a.H) or tuple(d_pooled.shape) != (a.B, E):
            raise TzkError("self_attn_pool_bwd: need lse [N, H] and d_pooled [B, E]")
        dq, dk, dv = (torch.empty((a.N, E), dtype=torch.float32, device=q.device) for _ in range(3))
        dsum = self._workspace("self_attn_pool_dsum", max(a.N * a.H, 1) * 4, q.device)
        a.lse, a.d_pooled, a.dsum = lse.data_ptr(), d_pooled.data_ptr(), dsum.data_ptr()
        a.dq, a.dk, a.dv = dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
        check(self._lib.tzk_self_attn_pool_bwd(ctypes.byref(a), self._seq_attn_grid(a, True), _stream()),
              "tzk_self_attn_pool_bwd")
        self.launches += int(a.B > 0)
        return dq, dk, dv

    def _jagged_pool_args(self, offsets, D: int, max_len: int, mean: bool):
        from ._lib import TzkJaggedPoolArgs

        _need(offsets, torch.int64, "offsets")
        a = TzkJaggedPoolArgs()
        a.B, a.D, a.max_len, a.mean = offsets.numel() - 1, int(D), int(max_len), int(bool(mean))
        a.offsets = offsets.data_ptr()
        return a

    def jagged_pool_fwd(self, seq, offsets, max_len: int, mean: bool):
        """seq [N, D] jagged rows -> out [B, D]: the sum (mean: over max(kept rows, 1)) of each sample's first
        max_len rows (0: all)."""
        _need(seq, torch.float32, "seq")
        a = self._jagged_pool_args(offsets, seq.shape[1], max_len, mean)
        a.N = seq.shape[0]
        out = torch.empty((a.B, a.D), dtype=torch.float32, device=seq.device)
        a.seq, a.out = seq.data_ptr(), out.data_ptr()
        check(self._lib.tzk_jagged_pool_fwd(ctypes.byref(a), self._grid(-(-max(a.B, 1) // 8), 8), _stream()),
              "tzk_jagged_pool_fwd")
        self.launches += int(a.B > 0)
        return out

    def jagged_pool_bwd(self, d_out, offsets, N: int, max_len: int, mean: bool):
        """d_out [B, D] -> d_seq [N, D] (0 on cropped rows)."""
        _need(d_out, torch.float32, "d_out")
        a = self._jagged_pool_args(offsets, d_out.shape[1], max_len, mean)
        a.N = int(N)
        d_seq = torch.empty((a.N, a.D), dtype=torch.float32, device=d_out.device)
        a.d_out, a.d_seq = d_out.data_ptr(), d_seq.data_ptr()
        check(self._lib.tzk_jagged_pool_bwd(ctypes.byref(a), self._grid(-(-max(a.B, 1) // 8), 8), _stream()),
              "tzk_jagged_pool_bwd")
        self.launches += int(a.B > 0)
        return d_seq

@dataclass
class ColPlan:
    """CSR description of a column gather-sum (K6): column c of the destination sums
    srcs[col_src[k]][:, col_srccol[k]] for k in [col_start[c], col_start[c+1])."""

    col_start: List[int]
    col_src: List[int]
    col_srccol: List[int]
    d_col_start: Optional[torch.Tensor] = None
    d_col_src: Optional[torch.Tensor] = None
    d_col_srccol: Optional[torch.Tensor] = None

    @property
    def C(self) -> int:
        return len(self.col_start) - 1

    def to(self, device) -> "ColPlan":
        self.d_col_start = torch.tensor(self.col_start, dtype=torch.int32, device=device)
        self.d_col_src = torch.tensor(self.col_src or [0], dtype=torch.int32, device=device)
        self.d_col_srccol = torch.tensor(self.col_srccol or [0], dtype=torch.int32, device=device)
        return self


_default: Optional[CudaKernels] = None


def default_kernels() -> CudaKernels:
    global _default
    if _default is None:
        _default = CudaKernels()
    return _default
