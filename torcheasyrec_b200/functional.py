"""Autograd-aware operators of the hot path, each a thin shell over one or two tzk kernels.

The compute backend is `CudaKernels` (kernels.py).  `use_backend()` exists so that the host-side logic
(sharding plans, all-to-all plumbing, regroup plans) can be unit-tested on a CPU box by *tests* that inject
their own checker backend; the package itself never provides one and every default path raises on CPU
tensors.
"""

import contextlib
import ctypes
import math
from typing import List, Optional, Sequence

import torch

from .kernels import ColPlan, default_kernels

_backend = None


def backend():
    return _backend if _backend is not None else default_kernels()


@contextlib.contextmanager
def use_backend(b):
    """Test hook: run host logic against an injected kernel backend."""
    global _backend
    prev, _backend = _backend, b
    try:
        yield
    finally:
        _backend = prev


def autocast_dtype(t: torch.Tensor) -> Optional[torch.dtype]:
    """The dtype torch.autocast casts to on `t`'s device type, or None when autocast is off there.

    Autocast never sees a custom autograd.Function, so every hand-written dense path asks this first.  Under autocast a
    path either keeps its fp32 kernel, where autocast itself would run that op in fp32 on the same inputs, or steps
    aside to the reference's torch formulation, which autocast then applies to (train_config.mixed_precision)."""
    dt = t.device.type
    if dt in ("cuda", "cpu") and torch.is_autocast_enabled(dt):
        return torch.get_autocast_dtype(dt)
    return None


def _rows_contig(t: torch.Tensor) -> torch.Tensor:
    if t.dim() == 2 and (t.shape[1] <= 1 or t.stride(1) == 1) and (t.shape[0] <= 1 or t.stride(0) >= t.shape[1]):
        return t
    return t.contiguous()


# ------------------------------------------------------------------------------------------------ K6
class _ColPlanCache:
    def __init__(self):
        self.cache = {}

    def get(self, key, build, device):
        k = (key, str(device))
        if k not in self.cache:
            self.cache[k] = build().to(device)
        return self.cache[k]


_plans = _ColPlanCache()


class _Regroup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, spec, *srcs):
        # spec: (src_widths, groups) with groups = tuple of tuples of (src, col, width)
        src_widths, groups = spec
        dev = srcs[0].device
        rows = srcs[0].shape[0]
        srcs_c = [_rows_contig(s) for s in srcs]
        outs = []
        for gi, g in enumerate(groups):
            def build(g=g):
                start, src, scol = [0], [], []
                for (s, c, w) in g:
                    for j in range(w):
                        src.append(s)
                        scol.append(c + j)
                        start.append(len(src))
                return ColPlan(start, src, scol)
            plan = _plans.get(("fwd", src_widths, groups, gi), build, dev)
            outs.append(backend().col_gather_sum(srcs_c, plan, rows))
        ctx.spec = spec
        ctx.dev = dev
        ctx.needs = [s.requires_grad for s in srcs]
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        src_widths, groups = ctx.spec
        rows = gouts[0].shape[0]
        g_c = [_rows_contig(g) for g in gouts]
        grads = [None]
        for si, width in enumerate(src_widths):
            if not ctx.needs[si]:
                grads.append(None)
                continue
            def build(si=si, width=width):
                contrib = [[] for _ in range(width)]
                for gi, g in enumerate(groups):
                    oc = 0
                    for (s, c, w) in g:
                        if s == si:
                            for j in range(w):
                                contrib[c + j].append((gi, oc + j))
                        oc += w
                start, src, scol = [0], [], []
                for lst in contrib:
                    for (gi, oc) in lst:
                        src.append(gi)
                        scol.append(oc)
                    start.append(len(src))
                return ColPlan(start, src, scol)
            plan = _plans.get(("bwd", src_widths, groups, si), build, ctx.dev)
            grads.append(backend().col_gather_sum(g_c, plan, rows))
        return tuple(grads)


def regroup(keyed_tensors, groups: Sequence[Sequence[str]]) -> List[torch.Tensor]:
    """KeyedTensor.regroup (tzrec/modules/embedding.py:972-976): per group, concat the named key columns.

    A group that is exactly one whole source tensor is returned as that tensor (no copy)."""
    where = {}
    for si, kt in enumerate(keyed_tensors):
        c = 0
        for k, n in zip(kt.keys(), kt.length_per_key()):
            where.setdefault(k, (si, c, n))
            c += n
    src_widths = tuple(kt.values().shape[1] for kt in keyed_tensors)
    spec_groups = []
    for g in groups:
        segs = []
        for k in g:
            s, c, n = where[k]
            if segs and segs[-1][0] == s and segs[-1][1] + segs[-1][2] == c:
                segs[-1] = (s, segs[-1][1], segs[-1][2] + n)  # merge adjacent columns
            else:
                segs.append((s, c, n))
        spec_groups.append(tuple(segs))
    # identity fast path
    outs: List[Optional[torch.Tensor]] = [None] * len(groups)
    todo = []
    for gi, segs in enumerate(spec_groups):
        if len(segs) == 1 and segs[0][1] == 0 and segs[0][2] == src_widths[segs[0][0]]:
            outs[gi] = keyed_tensors[segs[0][0]].values()
        else:
            todo.append(gi)
    if todo:
        res = _Regroup.apply((src_widths, tuple(spec_groups[gi] for gi in todo)),
                             *[kt.values() for kt in keyed_tensors])
        for gi, r in zip(todo, res):
            outs[gi] = r
    return outs


# ------------------------------------------------------------------------------------------------ K7
class _JaggedToPadded(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, offsets, T):
        ctx.save_for_backward(offsets)
        ctx.nnz = values.shape[0]
        return backend().jagged_to_padded(values.contiguous(), offsets, T)

    @staticmethod
    def backward(ctx, g):
        (offsets,) = ctx.saved_tensors
        return backend().padded_to_jagged(g.contiguous(), offsets, ctx.nnz), None, None


def jagged_to_padded_dense(values: torch.Tensor, offsets: torch.Tensor, T: int) -> torch.Tensor:
    if values.dim() == 1:
        return _JaggedToPadded.apply(values.unsqueeze(1), offsets, T).squeeze(2)
    return _JaggedToPadded.apply(values, offsets, T)


# ------------------------------------------------------------------------------------------------ K2
_perm_cache = {}


def kjt_permute(kjt, indices: List[int]):
    from .sparse import KeyedJaggedTensor

    B = kjt.stride()
    dev = kjt.values().device
    pk = (tuple(indices), str(dev))
    perm = _perm_cache.get(pk)
    if perm is None:      # cached: no host->device copy inside a captured step
        perm = _perm_cache[pk] = torch.tensor(indices, dtype=torch.int32, device=dev)
    new_len = backend().permute_lengths(kjt.lengths().contiguous(), perm, B)
    new_off = backend().lengths_to_offsets(new_len)
    lpk = kjt.length_per_key()
    out_nnz = sum(lpk[i] for i in indices)
    new_ids = backend().permute_ids(kjt.values(), kjt.offsets(), new_off, perm, B, out_nnz)
    w = kjt.weights_or_none()
    new_w = None if w is None else backend().permute_weights(w, kjt.offsets(), new_off, perm, B, out_nnz)
    out = KeyedJaggedTensor([kjt.keys()[i] for i in indices], new_ids, lengths=new_len, offsets=new_off, weights=new_w,
                            stride=B)
    out._length_per_key = [lpk[i] for i in indices]
    return out


# ------------------------------------------------------------------------------------------------ A7
class _FM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x2d, N, D):
        ctx.save_for_backward(x2d)
        ctx.nd = (N, D)
        return backend().fm_fwd(x2d, N, D)

    @staticmethod
    def backward(ctx, dy):
        (x2d,) = ctx.saved_tensors
        N, D = ctx.nd
        return backend().fm_bwd(x2d, _rows_contig(dy), N, D), None, None


def factorization_machine(feature: torch.Tensor) -> torch.Tensor:
    """[B, N, D] -> [B, D]  (tzrec/modules/fm.py:28-42).

    Under autocast an fp32 input keeps the kernel: sum and mul are on no lower-precision list (CUDA autocast runs sum in
    fp32, CPU autocast leaves both alone), so autocast computes the reference in fp32 too.  Any other input dtype takes
    the reference's torch formulation."""
    if autocast_dtype(feature) is not None and feature.dtype != torch.float32:
        s = torch.sum(feature, dim=1)
        return 0.5 * (s * s - torch.sum(feature * feature, dim=1))
    B, N, D = feature.shape
    return _FM.apply(_rows_contig(feature.reshape(B, N * D)), N, D)


# ------------------------------------------------------------------------------------------------ A9/A10
class _DotInteract(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dense, sparse, Ns, D, copy_dense, copy_sparse, pad_to=1, p_pad=0):
        dense_c = None if dense is None else _rows_contig(dense)
        sparse_c = _rows_contig(sparse)
        ctx.save_for_backward(dense_c, sparse_c)
        ctx.cfg = (Ns, D, copy_dense, copy_sparse, p_pad)
        return backend().dot_interact_fwd(dense_c, sparse_c, Ns, D, copy_dense, copy_sparse, pad_to, p_pad)

    @staticmethod
    def backward(ctx, d_out):
        dense, sparse = ctx.saved_tensors
        Ns, D, cd, cs, p_pad = ctx.cfg
        d_dense, d_sparse = backend().dot_interact_bwd(dense, sparse, _rows_contig(d_out), Ns, D, cd, cs, p_pad)
        return d_dense, d_sparse, None, None, None, None, None, None


_triu_cache = {}


def _torch_dot_interaction(features: torch.Tensor) -> torch.Tensor:
    """tzrec/modules/interaction.py:80-91 as stated there: bmm, then the strict upper triangle, row-major."""
    N = features.shape[1]
    key = (N, str(features.device))
    iu = _triu_cache.get(key)
    if iu is None:      # cached: no index build inside a captured step
        iu = _triu_cache[key] = torch.triu_indices(N, N, offset=1, device=features.device)
    z = torch.bmm(features, torch.transpose(features, 1, 2))
    return z[:, iu[0], iu[1]]


def _interact_rows_ok(t: torch.Tensor) -> bool:
    return (t.dtype == torch.float32 and t.dim() == 2 and (t.shape[1] <= 1 or t.stride(1) == 1)
            and (t.shape[0] <= 1 or t.stride(0) % 4 == 0) and t.data_ptr() % 16 == 0)


def dot_interact_usable(dense: Optional[torch.Tensor], sparse: torch.Tensor, Ns: int, D: int) -> bool:
    """True when the dot-interaction kernels (csrc/tzk_dense.cu) cover this call: fp32 [B, Ns*D] sparse and [B, D]
    dense (or None) with autocast off, 4 <= D <= 128 and D % 4 == 0, at most 64 features in all, every row contiguous
    and starting on a 16-B boundary, on a device the compute backend runs (CUDA; on the CPU only a test backend that
    implements the interaction kernels)."""
    if autocast_dtype(sparse) is not None or not (4 <= D <= 128 and D % 4 == 0) or Ns < 1:
        return False
    if Ns + (dense is not None) > 64 or not _interact_rows_ok(sparse) or sparse.shape[1] != Ns * D:
        return False
    if dense is not None and not (_interact_rows_ok(dense) and dense.shape[1] == D):
        return False
    return sparse.is_cuda or (_backend is not None and hasattr(_backend, "dot_interact_fwd"))


def dot_interaction(features: torch.Tensor) -> torch.Tensor:
    """InteractionArch.forward (tzrec/modules/interaction.py:80-91): [B,N,D] -> [B, N(N-1)/2].

    Under autocast, and for shapes outside dot_interact_usable, this is the reference's torch formulation (bmm is on
    autocast's lower-precision list)."""
    B, N, D = features.shape
    x = _rows_contig(features.reshape(B, N * D))
    if not dot_interact_usable(None, x, N, D):
        return _torch_dot_interaction(features)
    return _DotInteract.apply(None, x, N, D, False, False)


def dlrm_interaction(dense_feat: Optional[torch.Tensor], sparse_feat: torch.Tensor, num_sparse: int, dim: int,
                     with_dense: bool = True, with_sparse: bool = True, aligned: bool = False):
    """Fused DLRM.predict glue (tzrec/models/dlrm.py:113-131):
    cat([interaction(cat([dense[:,None,:], sparse.view(B,Ns,D)], 1)), dense, sparse], -1) in one pass.

    aligned=False -> the reference's exact column layout [P | dense | sparse].
    aligned=True  -> (tensor, in_map): zero columns are inserted after the P interaction terms and at the row end so
    that every block and every row starts on a 16-B boundary; `in_map` = [(src_col, dst_col, length), ...] tells the
    consuming Linear where the reference's columns live (dense_gemm.linear pads its weight accordingly).

    Under autocast, and for shapes outside dot_interact_usable (e.g. an embedding dim that is not a multiple of 4), this
    is the reference's torch formulation in the reference's layout (with aligned=True the map is None): autocast rounds
    the bmm to its dtype and the concatenations promote back to fp32, as in dlrm.py.  DLRM-Criteo under bf16 autocast has
    its own kernel (dense_gemm.InteractBf16Fn)."""
    if dense_feat is not None:
        dense_feat = _rows_contig(dense_feat)
    sparse_feat = _rows_contig(sparse_feat)
    if not dot_interact_usable(dense_feat, sparse_feat, num_sparse, dim):
        B = sparse_feat.shape[0]
        feat = sparse_feat.reshape(-1, num_sparse, dim)
        if dense_feat is not None:
            feat = torch.cat([dense_feat.unsqueeze(1), feat], dim=1)
        x = _torch_dot_interaction(feat)
        if with_dense and dense_feat is not None:
            x = torch.cat([x, dense_feat], dim=-1)
        if with_sparse:
            x = torch.cat([x, sparse_feat.reshape(B, -1)], dim=-1)
        return (x, None) if aligned else x
    if not aligned:
        return _DotInteract.apply(dense_feat, sparse_feat, num_sparse, dim, with_dense, with_sparse, 1, 0)
    n = num_sparse + (dense_feat is not None)
    P = n * (n - 1) // 2
    p_pad = (-P) % 4
    rest = (dim if (with_dense and dense_feat is not None) else 0) + (num_sparse * dim if with_sparse else 0)
    out = _DotInteract.apply(dense_feat, sparse_feat, num_sparse, dim, with_dense, with_sparse, 4, p_pad)
    return out, ((0, 0, P), (P, P + p_pad, rest))


# ------------------------------------------------------------------------------------------------ N3: jagged DIN
class _DinAttnInput(torch.autograd.Function):
    @staticmethod
    def forward(ctx, query, seq, offsets):
        q, k = _rows_contig(query), seq.contiguous()
        ctx.save_for_backward(q, k, offsets)
        return backend().din_attn_input_fwd(q, k, offsets)

    @staticmethod
    def backward(ctx, d_in):
        q, k, offsets = ctx.saved_tensors
        d_q, d_k = backend().din_attn_input_bwd(d_in.contiguous(), q, k, offsets)
        return d_q, d_k, None


class _JaggedSoftmaxWsum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores, seq, offsets, max_len):
        k = seq.contiguous()
        probs, out = backend().jagged_softmax_wsum_fwd(scores.contiguous(), k, offsets, max_len)
        ctx.save_for_backward(probs, k, offsets)
        ctx.max_len = max_len
        return out

    @staticmethod
    def backward(ctx, d_out):
        probs, k, offsets = ctx.saved_tensors
        d_s, d_k = backend().jagged_softmax_wsum_bwd(d_out.contiguous(), probs, k, offsets, ctx.max_len)
        return d_s, d_k, None, None


def _segments(offsets: torch.Tensor, n: int) -> torch.Tensor:
    """Sample index of each of the n jagged rows."""
    B = offsets.numel() - 1
    return torch.repeat_interleave(torch.arange(B, device=offsets.device), offsets[1:] - offsets[:-1], output_size=n)


def din_attn_input(query: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
    """[N, 4*Ds] input of DIN's attention MLP for jagged sequence rows: [q | k | q - k | q * k]
    (tzrec/modules/sequence.py:113-116 without the padded [B, T, Ds] broadcast).

    Under autocast fp32 inputs keep the kernel: pad, cat, sub and mul are on no lower-precision list, so autocast
    computes the reference in fp32 as the kernel does.  Other input dtypes take the torch formulation over the jagged
    rows."""
    if autocast_dtype(seq) is not None and (query.dtype != torch.float32 or seq.dtype != torch.float32):
        q = torch.nn.functional.pad(query, (0, seq.shape[1] - query.shape[1]))[_segments(offsets, seq.shape[0])]
        return torch.cat([q, seq, q - seq, q * seq], dim=-1)
    return _DinAttnInput.apply(query, seq, offsets)


def _torch_jagged_softmax_wsum(scores, seq, offsets, max_len: int, dtype) -> torch.Tensor:
    """tzrec/modules/sequence.py:124-128 under autocast, over jagged rows: softmax in fp32 (CUDA autocast's softmax is on
    its fp32 list; a CPU bf16 softmax also accumulates in fp32 and rounds once), then matmul on the lower-precision list:
    bf16 probabilities times bf16 rows, fp32 accumulation, one rounding of the result.  Padded positions of the
    reference carry probability exactly 0, so leaving them out changes only the summation order."""
    N, B = seq.shape[0], offsets.numel() - 1
    seg = _segments(offsets, N)
    s = scores.float()
    if max_len > 0:
        pos = torch.arange(N, device=seq.device) - offsets[:-1][seg]
        s = s.masked_fill(pos >= max_len, float("-inf"))
    m = torch.full((B,), float("-inf"), device=seq.device).scatter_reduce(0, seg, s.detach(), "amax")
    e = torch.exp(s - m[seg])
    z = torch.zeros(B, device=seq.device).index_add(0, seg, e)
    p = (e / z[seg]).to(dtype)
    out = torch.zeros((B, seq.shape[1]), device=seq.device).index_add(0, seg, p.float()[:, None] * seq.to(dtype).float())
    return out.to(dtype)


def jagged_softmax_weighted_sum(scores: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor,
                                max_len: int = 0) -> torch.Tensor:
    """[B, Ds]: per sample softmax over its (first max_len) scores, then the weighted sum of its rows
    (tzrec/modules/sequence.py:118-128; a sample without rows gives zeros like the masked padded version).

    Under autocast the weighted sum is a lower-precision matmul in the reference, so this takes the torch formulation
    (_torch_jagged_softmax_wsum) instead of the fp32 kernel."""
    dt = autocast_dtype(seq)
    if dt is not None:
        return _torch_jagged_softmax_wsum(scores, seq, offsets, int(max_len), dt)
    return _JaggedSoftmaxWsum.apply(scores, seq, offsets, int(max_len))


# ------------------------------------------------------------------------------------------------ WuKong layer
def wukong_usable(x: torch.Tensor, n: int, d: int, k: int, f: int, l: int) -> bool:
    """True when the fused WuKong kernels (csrc/tzk_wukong.cuh) cover this layer call: fp32 [B, n, d] input with
    n <= 64, d in {4, 8, 16, 32}, k <= 32, f, l >= 1 and f + l <= 64, autocast off, on a device the compute backend
    runs (CUDA; on the CPU only a test backend that implements the WuKong kernels)."""
    if autocast_dtype(x) is not None or x.dtype != torch.float32 or x.dim() != 3 or tuple(x.shape[1:]) != (n, d):
        return False
    if not (1 <= n <= 64 and d in (4, 8, 16, 32) and 1 <= k <= 32 and f >= 1 and l >= 1 and f + l <= 64):
        return False
    return x.is_cuda or (_backend is not None and hasattr(_backend, "wukong_mix_fwd"))


class _WuKongMix(torch.autograd.Function):
    """x -> (LayerNorm(n k)(X (X^T W_fmb)), base): the FMB's interaction and norm, and the LCB + residual."""

    @staticmethod
    def forward(ctx, x, w_fmb, gamma, beta, w_lcb, w_res, f):
        x = x.contiguous()
        ln_f, stats, base = backend().wukong_mix_fwd(x, w_fmb, gamma, beta, w_lcb, w_res, f)
        ctx.save_for_backward(x, w_fmb, gamma, w_lcb, w_res, stats)
        ctx.f = f
        return ln_f, base

    @staticmethod
    def backward(ctx, d_ln_f, d_base):
        x, w_fmb, gamma, w_lcb, w_res, stats = ctx.saved_tensors
        B, n, d = x.shape
        if d_ln_f is None:
            d_ln_f = x.new_zeros((B, n * w_fmb.shape[1]))
        if d_base is None:
            d_base = x.new_zeros((B, ctx.f + w_lcb.shape[1], d))
        dx, dwf, dg, db, dwl, dwr = backend().wukong_mix_bwd(x, w_fmb, gamma, w_lcb, w_res, ctx.f, stats,
                                                             d_ln_f.contiguous(), d_base.contiguous())
        return dx, dwf, dg, db, dwl, dwr, None


class _WuKongOut(torch.autograd.Function):
    """(fmb_out, base) -> LayerNorm(d)(concat(fmb, lcb) + residual)."""

    @staticmethod
    def forward(ctx, fmb_out, base, gamma, beta, f):
        fmb_out = fmb_out.contiguous()
        y, stats = backend().wukong_out_fwd(fmb_out, base, gamma, beta, f)
        ctx.save_for_backward(fmb_out, base, gamma, stats)
        ctx.f = f
        return y

    @staticmethod
    def backward(ctx, dy):
        fmb_out, base, gamma, stats = ctx.saved_tensors
        d_fmb, d_base, dg, db = backend().wukong_out_bwd(fmb_out, base, gamma, ctx.f, stats, dy.contiguous())
        return d_fmb, d_base, dg, db, None


def wukong_mix(x: torch.Tensor, w_fmb: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, w_lcb: torch.Tensor,
               w_res: Optional[torch.Tensor], f: int):
    """Fused first half of a WuKong layer (csrc/tzk_wukong.cuh mix_fwd / mix_bwd): x [B, n, d] ->
    (LayerNorm(X (X^T w_fmb)) [B, n k], base [B, f + l, d]) where base holds the residual (w_res^T X, or X when w_res is
    None) and, on rows >= f, lcb + residual.  The caller checks wukong_usable first."""
    return _WuKongMix.apply(x, w_fmb, gamma, beta, w_lcb, w_res, f)


def wukong_out(fmb_out: torch.Tensor, base: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, f: int):
    """Fused end of a WuKong layer (csrc/tzk_wukong.cuh out_fwd / out_bwd): LayerNorm(d) with affine of base with
    fmb_out [B, f d] added to its first f rows -> [B, f + l, d]."""
    return _WuKongOut.apply(fmb_out, base, gamma, beta, f)


def torch_wukong_interaction(x: torch.Tensor, w_fmb: torch.Tensor) -> torch.Tensor:
    """FactorizationMachineBlock's interaction as the reference states it (tzrec/modules/interaction.py:314-317):
    X (X^T W) flattened to [B, n k]."""
    t = torch.matmul(x.permute(0, 2, 1), w_fmb)
    return torch.matmul(x, t).reshape(x.shape[0], -1)


def torch_linear_compress(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """LinearCompressBlock.forward (tzrec/modules/interaction.py:255-264): W^T X as [B, l, d]."""
    return (x.permute(0, 2, 1) @ w).permute(0, 2, 1)


# ------------------------------------------------------------------------------------------------ MaskNet
MASKNET_MAX_WIDTH = 1024     # csrc/tzk_masknet.cuh kMaxWidth: pad4(E) and H
MASKNET_MAX_BLOCKS = 8


def _pad4(n: int) -> int:
    return (n + 3) // 4 * 4


def masknet_usable(e: torch.Tensor, E: int, H: int, n_blocks: int, use_parallel: bool) -> bool:
    """True when the fused MaskNet path (csrc/tzk_masknet.cuh around cuBLASLt GEMMs) covers this module call: parallel
    blocks, fp32 [B, E] input with pad4(E) <= 1024, 4 <= H <= 1024 and H % 4 == 0, 1 <= n_blocks <= 8, autocast off, on
    CUDA with the dense GEMM library loaded and TF32 off (on the CPU only a test backend that implements the MaskNet
    kernels)."""
    if not use_parallel or autocast_dtype(e) is not None or e.dtype != torch.float32 or e.dim() != 2:
        return False
    if e.shape[1] != E or not (1 <= E and _pad4(E) <= MASKNET_MAX_WIDTH and 4 <= H <= MASKNET_MAX_WIDTH and H % 4 == 0
                               and 1 <= n_blocks <= MASKNET_MAX_BLOCKS):
        return False
    if e.is_cuda:
        from . import dense_gemm

        return _backend is None and dense_gemm.available() and not torch.backends.cuda.matmul.allow_tf32
    return _backend is not None and hasattr(_backend, "masknet_mask_fwd")


class _MaskNetParallel(torch.autograd.Function):
    """e [B, E] -> hidden [B, nb H] of MaskNetModule's parallel blocks (tzrec/modules/masknet.py:77-85, 142-151).

    Every GEMM operand and result has a row pitch that is a multiple of 4 floats: E travels as Ep = pad4(E) and the
    aggregation width A as Ap = pad4(A), with zero columns and zero weight rows / columns (their gradients dropped).
      h  = ReLU(e W1cat^T + b1cat)        one GEMM over all blocks, N = nb Ap, then bias_act
      m_i = h_i W2_i^T                    into m [B, nb Ep], block i at columns i Ep
      v, stats = mask_fwd(e, m, b2)       LN(e) * (m_i + b2_i)
      z_i = v_i W3_i^T                    into z [B, nb H]
      hidden, stats2 = ffn_fwd(z, b3)     ReLU(LN_H(z_i + b3_i)) in block i's slot of hidden
    The backward mirrors it; the input gradient is de_ln (mask_bwd) + dh W1cat as one GEMM with beta = 1."""

    @staticmethod
    def forward(ctx, e, ln_w, ln_b, *params):
        from . import dense_gemm

        K = backend()
        nb = len(params) // 8
        w1s, b1s, w2s, b2s, w3s, b3s, gs, bs = (params[j::8] for j in range(8))
        B, E = e.shape
        A, H = w1s[0].shape[0], w3s[0].shape[0]
        Ep, Ap = _pad4(E), _pad4(A)
        e_p = e.new_zeros((B, Ep))
        e_p[:, :E] = e
        w1cat = e.new_zeros((nb * Ap, Ep))
        b1cat = e.new_zeros((nb * Ap,))
        w2p = e.new_zeros((nb, Ep, Ap))
        w3p = e.new_zeros((nb, H, Ep))
        for i in range(nb):
            w1cat[i * Ap:i * Ap + A, :E] = w1s[i]
            b1cat[i * Ap:i * Ap + A] = b1s[i]
            w2p[i, :E, :A] = w2s[i]
            w3p[i, :, :E] = w3s[i]
        b2cat, b3cat = torch.cat(b2s).contiguous(), torch.cat(b3s).contiguous()
        gcat, bcat = torch.cat(gs).contiguous(), torch.cat(bs).contiguous()
        ln_w, ln_b = ln_w.contiguous(), ln_b.contiguous()

        h = dense_gemm.gemm(e_p, False, w1cat, True)
        if h.is_cuda:
            K.bias_act(h, b1cat, True)
        else:
            h.add_(b1cat).relu_()
        m = e.new_empty((B, nb * Ep))
        for i in range(nb):
            dense_gemm.gemm(h[:, i * Ap:(i + 1) * Ap], False, w2p[i], True, out=m[:, i * Ep:(i + 1) * Ep])
        v, stats = K.masknet_mask_fwd(e_p, m, b2cat, ln_w, ln_b, E, nb)
        z = e.new_empty((B, nb * H))
        for i in range(nb):
            dense_gemm.gemm(v[:, i * Ep:(i + 1) * Ep], False, w3p[i], True, out=z[:, i * H:(i + 1) * H])
        hidden, stats2 = K.masknet_ffn_fwd(z, b3cat, gcat, bcat, nb)
        ctx.save_for_backward(e_p, h, m, v, z, stats, stats2, w1cat, w2p, w3p, b2cat, b3cat, gcat, bcat, ln_w, ln_b)
        ctx.dims = (nb, E, A, H)
        return hidden

    @staticmethod
    def backward(ctx, d_hidden):
        from . import dense_gemm

        K = backend()
        e_p, h, m, v, z, stats, stats2, w1cat, w2p, w3p, b2cat, b3cat, gcat, bcat, ln_w, ln_b = ctx.saved_tensors
        nb, E, A, H = ctx.dims
        B, Ep = e_p.shape
        Ap = h.shape[1] // nb
        dz, dg, dbeta, db3 = K.masknet_ffn_bwd(z, b3cat, gcat, bcat, stats2, d_hidden.contiguous(), nb)
        dv = e_p.new_empty((B, nb * Ep))
        dw3 = []
        for i in range(nb):
            dz_i = dz[:, i * H:(i + 1) * H]
            dense_gemm.gemm(dz_i, False, w3p[i], False, out=dv[:, i * Ep:(i + 1) * Ep])
            dw3.append(dense_gemm.gemm(dz_i, True, v[:, i * Ep:(i + 1) * Ep], False)[:, :E])
        dm, de_p, db2, dln_w, dln_b = K.masknet_mask_bwd(e_p, m, b2cat, ln_w, ln_b, stats, dv, E, nb)
        dh = e_p.new_empty((B, nb * Ap))
        dw2 = []
        for i in range(nb):
            dm_i = dm[:, i * Ep:(i + 1) * Ep]
            dense_gemm.gemm(dm_i, False, w2p[i], False, out=dh[:, i * Ap:(i + 1) * Ap])
            dw2.append(dense_gemm.gemm(dm_i, True, h[:, i * Ap:(i + 1) * Ap], False)[:E, :A])
        dh.mul_(h > 0)                                   # ReLU backward of the first mask-generator layer
        db1 = dh.sum(0)
        dw1 = dense_gemm.gemm(dh, True, e_p, False)
        dense_gemm.gemm(dh, False, w1cat, False, out=de_p, beta=1.0)
        grads = []
        for i in range(nb):
            grads += [dw1[i * Ap:i * Ap + A, :E], db1[i * Ap:i * Ap + A], dw2[i], db2[i * E:(i + 1) * E], dw3[i],
                      db3[i], dg[i], dbeta[i]]
        return (de_p[:, :E], dln_w, dln_b, *grads)


def masknet_parallel(e: torch.Tensor, ln_w: torch.Tensor, ln_b: torch.Tensor, blocks: Sequence[Sequence[torch.Tensor]]):
    """Fused MaskNetModule body in parallel mode: e [B, E] -> concat_i MaskBlock_i(LN(e), e) [B, nb H].  `blocks` holds
    per block (W1, b1, W2, b2, W3, b3, gamma, beta) of mask_generator.0, mask_generator.2, ffn.0 and ffn.1.  The caller
    checks masknet_usable first."""
    return _MaskNetParallel.apply(e, ln_w, ln_b, *[p for blk in blocks for p in blk])


# ------------------------------------------------------------------------------------------------ PLE gates
PLE_MAX_GATES = 9             # csrc/tzk_ple.cuh: T <= 8 task gates + the shared gate
PLE_MAX_EXPERTS = 64
PLE_MAX_GATE_EXPERTS = 32
PLE_MAX_WIDTH = 1024          # H and K
PLE_MAX_WEIGHT_FLOATS = 20480  # sum_g E_g K_g, the gate weights held in shared memory


def ple_gate_usable(inputs: Sequence[torch.Tensor], gate_input: Sequence[int], weights: Sequence[torch.Tensor],
                    experts: Sequence[torch.Tensor], gate_experts: Sequence[Sequence[int]]) -> bool:
    """True when the fused gate kernels (csrc/tzk_ple.cuh) cover this extraction layer: fp32 2-D tensors, autocast off,
    at most 9 gates over at most 64 experts of one [B, H] shape with 1 <= H <= 1024, each gate over 1..32 distinct
    experts and an input of width 1 <= K <= 1024, sum_g E_g K_g <= 20480, on CUDA (on the CPU only a test backend that
    implements the PLE kernels)."""
    t = experts[0] if len(experts) else None
    if t is None or autocast_dtype(t) is not None:
        return False
    if any(x.dtype != torch.float32 or x.dim() != 2 or x.device != t.device
           for x in (*inputs, *experts, *weights)):
        return False
    B, H = t.shape
    if any(tuple(e.shape) != (B, H) for e in experts) or any(x.shape[0] != B for x in inputs):
        return False
    if not (1 <= len(gate_input) <= PLE_MAX_GATES and len(experts) <= PLE_MAX_EXPERTS and 1 <= H <= PLE_MAX_WIDTH
            and all(1 <= x.shape[1] <= PLE_MAX_WIDTH for x in inputs)):
        return False
    total = 0
    for g, ids in enumerate(gate_experts):
        K = inputs[gate_input[g]].shape[1]
        if not (1 <= len(ids) <= PLE_MAX_GATE_EXPERTS and len(set(ids)) == len(ids)
                and tuple(weights[g].shape) == (len(ids), K)):
            return False
        total += len(ids) * K
    if total > PLE_MAX_WEIGHT_FLOATS:
        return False
    return t.is_cuda or (_backend is not None and hasattr(_backend, "ple_gate_fwd"))


class _PleGates(torch.autograd.Function):
    """Every gate of one extraction layer: y_g = softmax(x_g W_g^T + b_g) @ stack(experts of g), as [n_gates, B, H]."""

    @staticmethod
    def forward(ctx, spec, *tensors):
        gate_input, gate_experts, n_in, n_exp = spec
        G = len(gate_input)
        inputs = [x.contiguous() for x in tensors[:n_in]]
        weights = [w.contiguous() for w in tensors[n_in:n_in + G]]
        biases = [b.contiguous() for b in tensors[n_in + G:n_in + 2 * G]]
        experts = [e.contiguous() for e in tensors[n_in + 2 * G:]]
        y, p = backend().ple_gate_fwd(inputs, gate_input, weights, biases, experts, gate_experts)
        ctx.save_for_backward(*inputs, *weights, *biases, *experts, p)
        ctx.spec = spec
        return y

    @staticmethod
    def backward(ctx, dy):
        gate_input, gate_experts, n_in, n_exp = ctx.spec
        G = len(gate_input)
        saved = ctx.saved_tensors
        inputs, weights = list(saved[:n_in]), list(saved[n_in:n_in + G])
        biases, experts, p = list(saved[n_in + G:n_in + 2 * G]), list(saved[n_in + 2 * G:-1]), saved[-1]
        d_inputs, d_experts, dW, db = backend().ple_gate_bwd(inputs, gate_input, weights, biases, experts,
                                                             gate_experts, p, dy.contiguous())
        return (None, *d_inputs, *dW, *db, *d_experts.unbind(0))


def ple_gates(inputs: Sequence[torch.Tensor], gate_input: Sequence[int], weights: Sequence[torch.Tensor],
              biases: Sequence[torch.Tensor], experts: Sequence[torch.Tensor],
              gate_experts: Sequence[Sequence[int]]) -> List[torch.Tensor]:
    """Fused gates of one PLE extraction layer (csrc/tzk_ple.cuh): gate g reads inputs[gate_input[g]] through the
    Linear (weights[g], biases[g]) and mixes experts[gate_experts[g]] in that order -> [y_g [B, H] per gate].  The
    caller checks ple_gate_usable first."""
    spec = (tuple(gate_input), tuple(tuple(ids) for ids in gate_experts), len(inputs), len(experts))
    y = _PleGates.apply(spec, *inputs, *weights, *biases, *experts)
    return list(y.unbind(0))


def torch_ple_gate(selector: torch.Tensor, experts: Sequence[torch.Tensor], gate: torch.nn.Module) -> torch.Tensor:
    """ExtractionNet._gate_forward (tzrec/modules/extraction_net.py:93-105): the reference's torch formulation."""
    vec = torch.stack(list(experts), dim=1)
    g = torch.softmax(gate(selector), dim=1).unsqueeze(1)
    return torch.matmul(g, vec).squeeze(1)


# ------------------------------------------------------------------------------------------------ PEPNet gates
PEPNET_MAX_TASKS = 8           # csrc/tzk_pepnet.cuh: one segment per task in one launch
PEPNET_MAX_WIDTH = 1024        # N of a segment


def pepnet_usable(main: torch.Tensor, other: torch.Tensor, gate_hidden: Sequence[int], widths: Sequence[int],
                  n_tasks: int = 1, activation: Optional[str] = None) -> bool:
    """True when the fused PEPNet path covers an EPNet (activation None: identity product, `other` the domain input) or
    a PPNet (`activation` its ppnet_activation, `other` the uia input): fp32 2-D inputs, autocast off, the gate input
    width other + main, every gate hidden width and every product width a multiple of 4, product widths <= 1024, 1 <=
    n_tasks <= 8, activation nn.ReLU (PPNet), on CUDA with the dense GEMM library loaded and TF32 off (on the CPU only
    a test backend that implements the PEPNet kernels)."""
    if autocast_dtype(main) is not None or activation not in (None, "nn.ReLU"):
        return False
    if any(t.dtype != torch.float32 or t.dim() != 2 or t.device != main.device for t in (main, other)):
        return False
    if other.shape[0] != main.shape[0] or (other.shape[1] + main.shape[1]) % 4 != 0:
        return False
    if not (1 <= n_tasks <= PEPNET_MAX_TASKS and all(h >= 4 and h % 4 == 0 for h in gate_hidden)
            and all(4 <= n <= PEPNET_MAX_WIDTH and n % 4 == 0 for n in widths)):
        return False
    if main.is_cuda:
        from . import dense_gemm

        return _backend is None and dense_gemm.available() and not torch.backends.cuda.matmul.allow_tf32
    return _backend is not None and hasattr(_backend, "pepnet_gate_fwd")


def _relu_bwd_colsum(dh: torch.Tensor, h: torch.Tensor):
    """(dh * (h > 0), its column sums) of a [B, N] layer, N % 4 == 0: act_bwd_colsum on column blocks of 256, 128, ...,
    4 (the widths it covers), into one [B, N] buffer."""
    if not dh.is_cuda:
        d = dh * (h > 0)
        return d, d.sum(0)
    K = backend()
    out = torch.empty_like(dh)
    sums, c, N = [], 0, dh.shape[1]
    while c < N:
        w = 256
        while w > N - c:
            w //= 2
        _, s = K.act_bwd_colsum(dh[:, c:c + w], h[:, c:c + w], True, out=out[:, c:c + w])
        sums.append(s)
        c += w
    return out, torch.cat(sums)


class _PepnetGateHidden(torch.autograd.Function):
    """Every GateNU of an EPNet or PPNet up to its sigmoid (tzrec/modules/personalized_net.py GateNU.dense_layers
    0..2), on the one gate input G = [other | main.detach()] (formed once, not per task):
      h = ReLU(G W1cat^T + b1cat)        one GEMM over every gate, then bias_act
      z_k = h_k W2_k^T                   one GEMM per gate, into column slot place[k] of output group place[k][0]
    The second layers' biases and the sigmoid belong to the product (_PepnetProduct).  Backward: dh_k = dz_k W2_k, the
    ReLU backward and db1 with act_bwd_colsum, dW1cat = dh^T G and d_other = dh W1cat[:, :U] as one GEMM each."""

    @staticmethod
    def forward(ctx, spec, other, main, *params):
        from . import dense_gemm

        K = backend()
        groups, place = spec
        G = len(place)
        w1s, b1s, w2s = params[:G], params[G:2 * G], params[2 * G:]
        g_in = torch.cat([other, main], dim=1)
        w1cat, b1cat = torch.cat(w1s).contiguous(), torch.cat(b1s).contiguous()
        h = dense_gemm.gemm(g_in, False, w1cat, True)
        if h.is_cuda:
            K.bias_act(h, b1cat, True)
        else:
            h.add_(b1cat).relu_()
        B = g_in.shape[0]
        zs = [g_in.new_empty((B, w)) for w in groups]
        off = 0
        for k in range(G):
            (grp, col), a, n = place[k], w1s[k].shape[0], w2s[k].shape[0]
            dense_gemm.gemm(h[:, off:off + a], False, w2s[k], True, out=zs[grp][:, col:col + n])
            off += a
        ctx.save_for_backward(g_in, h, w1cat, *w2s)
        ctx.spec, ctx.U = spec, other.shape[1]
        return tuple(zs)

    @staticmethod
    def backward(ctx, *dzs):
        from . import dense_gemm

        g_in, h, w1cat, *w2s = ctx.saved_tensors
        groups, place = ctx.spec
        dh = torch.empty_like(h)
        dw2, hidden, off = [], [], 0
        for k, w2 in enumerate(w2s):
            (grp, col), a, n = place[k], w2.shape[1], w2.shape[0]
            dz = _rows_contig(dzs[grp])[:, col:col + n]
            dense_gemm.gemm(dz, False, w2, False, out=dh[:, off:off + a])
            dw2.append(dense_gemm.gemm(dz, True, h[:, off:off + a], False))
            hidden.append(a)
            off += a
        dh, db1 = _relu_bwd_colsum(dh, h)
        dw1 = dense_gemm.gemm(dh, True, g_in, False)
        d_other = dense_gemm.gemm(dh, False, w1cat[:, :ctx.U], False) if ctx.needs_input_grad[1] else None
        dw1s, db1s, off = [], [], 0
        for a in hidden:
            dw1s.append(dw1[off:off + a])
            db1s.append(db1[off:off + a])
            off += a
        return (None, d_other, None, *dw1s, *db1s, *dw2)


class _PepnetProduct(torch.autograd.Function):
    """y_i = act(x_i + bx_i) * gamma sigmoid(z_i + bz_i) for T segments of width N side by side in y [B, T N]
    (csrc/tzk_pepnet.cuh, one launch each way).  x_i is inputs[0] itself (EPNet: no weights, identity), the i-th slot
    of one GEMM of the shared input against the stacked weights (PPNet depth 0), or one GEMM per task input (deeper
    depths).  z [B, T N] is _PepnetGateHidden's output group of this depth."""

    @staticmethod
    def forward(ctx, spec, z, *tensors):
        from . import dense_gemm

        n_in, T, relu, gamma = spec
        inputs, rest = tensors[:n_in], tensors[n_in:]
        has_w = len(rest) == 3 * T
        ws, bs, bzs = (rest[:T], rest[T:2 * T], rest[2 * T:]) if has_w else ((), (None,) * T, rest)
        B, N = z.shape[0], z.shape[1] // T
        z = _rows_contig(z)
        if not has_w:
            x = _rows_contig(inputs[0])
        elif n_in == 1:
            x = dense_gemm.gemm(inputs[0], False, torch.cat(ws), True)
        else:
            x = z.new_empty((B, T * N))
            for i in range(T):
                dense_gemm.gemm(inputs[i], False, ws[i], True, out=x[:, i * N:(i + 1) * N])
        y = z.new_empty((B, T * N))
        backend().pepnet_gate_fwd([(x[:, i * N:(i + 1) * N], bs[i], z[:, i * N:(i + 1) * N], bzs[i],
                                    y[:, i * N:(i + 1) * N], relu, gamma) for i in range(T)])
        ctx.save_for_backward(x, z, *inputs, *ws, *[b for b in bs if b is not None], *bzs)
        ctx.spec, ctx.has_w = spec, has_w
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import dense_gemm

        n_in, T, relu, gamma = ctx.spec
        x, z, *rest = ctx.saved_tensors
        inputs = rest[:n_in]
        ws, bs, bzs = (rest[n_in:n_in + T], rest[n_in + T:n_in + 2 * T], rest[n_in + 2 * T:]) if ctx.has_w \
            else ((), (None,) * T, rest[n_in:])
        N = z.shape[1] // T
        dy = _rows_contig(dy)
        dx, dz = torch.empty_like(x), torch.empty_like(z)
        cols = [slice(i * N, (i + 1) * N) for i in range(T)]
        sums = backend().pepnet_gate_bwd([(x[:, c], bs[i], z[:, c], bzs[i], None, relu, gamma) for i, c in enumerate(cols)],
                                         [dy[:, c] for c in cols], [dx[:, c] for c in cols], [dz[:, c] for c in cols])
        dbzs = [s[1] for s in sums]
        if not ctx.has_w:
            return (None, dz, dx, *dbzs)
        if n_in == 1:
            d_in = [dense_gemm.gemm(dx, False, torch.cat(ws), False)]
            dw = dense_gemm.gemm(dx, True, inputs[0], False)
            dws = [dw[c] for c in cols]
        else:
            d_in = [dense_gemm.gemm(dx[:, c], False, ws[i], False) for i, c in enumerate(cols)]
            dws = [dense_gemm.gemm(dx[:, c], True, inputs[i], False) for i, c in enumerate(cols)]
        return (None, dz, *d_in, *dws, *[s[0] for s in sums], *dbzs)


def pepnet_gate_hidden(other: torch.Tensor, main: torch.Tensor, gates, groups: Sequence[int], place) -> List[torch.Tensor]:
    """Fused first layers of the GateNUs `gates` (modules with dense_layers.0 / .2) on [other | main.detach()]:
    -> one [B, groups[g]] tensor per output group, gate k's pre-bias second layer at place[k] = (group, column).  The
    caller checks pepnet_usable first."""
    l1 = [g.dense_layers[0] for g in gates]
    params = [m.weight for m in l1] + [m.bias for m in l1] + [g.dense_layers[2].weight for g in gates]
    spec = (tuple(groups), tuple(tuple(p) for p in place))
    return list(_PepnetGateHidden.apply(spec, other, main.detach(), *params))


def pepnet_product(z: torch.Tensor, gates, gamma: float, inputs: Sequence[torch.Tensor], linears=(),
                   relu: bool = False) -> torch.Tensor:
    """Fused GateNU product of T = len(gates) segments side by side: [B, T N] with slot i = act(x_i + b_i) *
    gamma sigmoid(z_i + gates[i].dense_layers.2.bias), x_i = inputs[0] (no linears), inputs[0] through linears[i]
    (one shared input) or inputs[i] through linears[i].  The caller checks pepnet_usable first."""
    T = len(gates)
    params = ([m.weight for m in linears] + [m.bias for m in linears]) if linears else []
    params += [g.dense_layers[2].bias for g in gates]
    return _PepnetProduct.apply((len(inputs), T, bool(relu), float(gamma)), z, *inputs, *params)


# --------------------------------------------------------------------------------------------------------
# JRC loss (tzrec/loss/jrc_loss.py; csrc/tzk_jrc.cuh)
# --------------------------------------------------------------------------------------------------------
def torch_jrc_loss(logits: torch.Tensor, labels: torch.Tensor, session_ids: torch.Tensor, alpha: float,
                   reduction: str = "mean") -> torch.Tensor:
    """The JRC loss in O(B) torch ops: per sample alpha ce_i + (1 - alpha) ge_i, with ge_i the log-softmax of the
    sample's own logit of its class against the same-class logits of the other class's samples of its session.
    `reduction` "none": the [B] per-sample losses; "mean": their mean, NaN when the batch lacks a positive or a negative
    (as the reference's empty cross-entropy mean times 0), with the gradient of the finite terms.  A label outside
    {0, 1} gives a NaN term where the reference raises.  torch.unique reads the number of sessions on the host."""
    logits = logits.float()
    l0, l1 = logits[:, 0], logits[:, 1]
    y = labels.float()
    pos, neg = y == 1, y == 0
    _, inv = torch.unique(session_ids, return_inverse=True)
    U = int(inv.max()) + 1 if inv.numel() else 0

    def side(x, member):
        # per session: (max, sum exp(x - max)) over the members; the shift is a constant for autograd
        xd = torch.where(member, x.detach(), torch.full_like(x, float("-inf")))
        M = torch.full((U,), float("-inf"), dtype=x.dtype, device=x.device).scatter_reduce(0, inv, xd, "amax")
        Ms = torch.where(torch.isfinite(M), M, torch.zeros_like(M))
        xs = torch.where(member, x, Ms[inv])
        S = torch.zeros(U, dtype=x.dtype, device=x.device).index_add(0, inv, torch.exp(xs - Ms[inv]) * member)
        return M[inv], S[inv]

    M1, S1 = side(l1, neg)                 # the negatives' l1, against which a positive competes
    M0, S0 = side(l0, pos)                 # the positives' l0, against which a negative competes
    x = torch.where(pos, l1, l0)
    M, S = torch.where(pos, M1, M0), torch.where(pos, S1, S0)
    m = torch.maximum(x.detach(), M)
    ge = m - x + torch.log(torch.exp(x - m) + S * torch.exp(M - m))
    invalid = torch.where(pos | neg, torch.zeros_like(y), torch.full_like(y, float("nan")))
    ce = torch.logsumexp(logits, dim=1) - x + invalid
    loss = alpha * ce + (1.0 - alpha) * ge
    if reduction == "none":
        return loss
    nan_unless_both = torch.where(pos.any() & neg.any(), 0.0, float("nan")).to(loss.dtype)
    return loss.mean() + nan_unless_both


class _JrcLoss(torch.autograd.Function):
    """The loss and d loss / d logits in one tzk_jrc_loss call; the backward scales the saved gradient."""

    @staticmethod
    def forward(ctx, logits, labels, session_ids, weights, alpha, key_bits):
        loss, dlogits = backend().jrc_loss(_rows_contig(logits), labels, session_ids, weights, alpha, key_bits)
        ctx.save_for_backward(dlogits)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None, None, None, None


def jrc_usable(logits: torch.Tensor) -> bool:
    """True when tzk_jrc_loss computes the loss: 2-D [B, 2] logits on CUDA (on the CPU only a test backend that
    implements it)."""
    if logits.dim() != 2 or logits.shape[1] != 2:
        return False
    if logits.is_cuda:
        return _backend is None or hasattr(_backend, "jrc_loss")
    return _backend is not None and hasattr(_backend, "jrc_loss")


def jrc_loss(logits: torch.Tensor, labels: torch.Tensor, session_ids: torch.Tensor, alpha: float,
             weights: Optional[torch.Tensor] = None, key_bits: int = 64) -> torch.Tensor:
    """Scalar JRC loss: the mean of the per-sample losses (weights None, with the reference's NaN for a batch without a
    positive or a negative) or the mean of the per-sample losses times `weights` [B].  The logits are taken in fp32, as
    autocast runs cross_entropy.  session_ids must lie in [0, 2^key_bits).  Device work only on the fused path
    (capturable); otherwise torch_jrc_loss, which reads the session count on the host."""
    logits = logits.float()
    if jrc_usable(logits):
        y = labels.to(torch.float32).contiguous()
        w = None if weights is None else weights.to(torch.float32).expand(logits.shape[0]).contiguous()
        return _JrcLoss.apply(logits, y, session_ids.to(torch.int64).contiguous(), w, float(alpha), int(key_bits))
    if weights is None:
        return torch_jrc_loss(logits, labels, session_ids, alpha, "mean")
    return torch.mean(torch_jrc_loss(logits, labels, session_ids, alpha, "none") * weights)


# --------------------------------------------------------------------------------------------------------
# RocketLaunching head (tzrec/models/rocket_launching.py; csrc/tzk_rocket.cuh)
# --------------------------------------------------------------------------------------------------------
ROCKET_MAX_CLASSES = 8        # csrc/tzk_rocket.cuh: the logits of a sample stay in registers
ROCKET_MAX_PAIRS = 8          # similarity pairs in one launch
ROCKET_MAX_WIDTH = 1024       # hidden and pair widths
ROCKET_COSINE, ROCKET_EUCLID = 0, 1


def rocket_head_usable(hiddens: Sequence[torch.Tensor], num_class: int, pair_widths: Sequence[int]) -> bool:
    """True when tzk_rocket_head covers the heads over `hiddens` (light first) with `num_class` outputs and similarity
    pairs of `pair_widths`: fp32 2-D hidden layers, autocast and TF32 off, 2 <= num_class <= 8, every hidden and pair
    width a multiple of 4 from 4 to 1024, at most 8 pairs; on CUDA (on the CPU only a test backend that implements the
    kernels)."""
    t = hiddens[0]
    if autocast_dtype(t) is not None or not 2 <= num_class <= ROCKET_MAX_CLASSES or len(pair_widths) > ROCKET_MAX_PAIRS:
        return False
    if any(h.dtype != torch.float32 or h.dim() != 2 or h.device != t.device for h in hiddens):
        return False
    if not all(4 <= w <= ROCKET_MAX_WIDTH and w % 4 == 0 for w in [h.shape[1] for h in hiddens] + list(pair_widths)):
        return False
    if t.is_cuda:
        return _backend is None and not torch.backends.cuda.matmul.allow_tf32
    return _backend is not None and hasattr(_backend, "rocket_head_fwd")


class _RocketHead(torch.autograd.Function):
    """Both heads' Linear + softmax and every loss of RocketLaunching in one tzk_rocket_head_fwd call, their gradients
    in one tzk_rocket_head_bwd call.  Outputs: logits and probs of every head (not differentiable), then the loss
    vector [CE light, CE booster, hint, sim_0, ...] (empty without labels)."""

    @staticmethod
    def forward(ctx, spec, labels, *tensors):
        n_heads, n_pairs, eps, sim = spec
        heads = [tuple(tensors[3 * e:3 * e + 3]) for e in range(n_heads)]
        rest = tensors[3 * n_heads:]
        pairs = [(rest[2 * k], rest[2 * k + 1]) for k in range(n_pairs)]
        logits, probs, losses, stats = backend().rocket_head_fwd(heads, labels, eps, pairs, sim)
        if losses is None:
            losses = logits[0].new_empty(0)
        ctx.mark_non_differentiable(*logits, *probs)
        ctx.save_for_backward(labels, stats, losses, *logits, *probs, *tensors)
        ctx.spec = spec
        return (*logits, *probs, losses)

    @staticmethod
    def backward(ctx, *grads):
        n_heads, n_pairs, eps, sim = ctx.spec
        labels, stats, losses, *rest = ctx.saved_tensors
        logits, probs, tensors = rest[:n_heads], rest[n_heads:2 * n_heads], rest[2 * n_heads:]
        heads = [tuple(tensors[3 * e:3 * e + 3]) for e in range(n_heads)]
        pr = tensors[3 * n_heads:]
        pairs = [(pr[2 * k], pr[2 * k + 1]) for k in range(n_pairs)]
        dlosses = grads[-1].to(torch.float32).contiguous()
        dhs, dlights, dparams = backend().rocket_head_bwd(heads, logits, probs, labels, eps, pairs, sim, stats, losses,
                                                          dlosses)
        out = [None, None]
        for dh, (dw, db) in zip(dhs, dparams):
            out += [dh, dw, db]
        for dl in dlights:
            out += [dl, None]
        return tuple(out)


def rocket_head(heads, labels: Optional[torch.Tensor], eps: float = 0.0, pairs=(), sim: int = ROCKET_COSINE):
    """heads [(h [B, H], weight [C, H], bias [C])]: the light head, then optionally the booster head; labels [B] (class
    indices) or None; pairs [(light [B, d], booster [B, d])], the booster side taken as detached.  -> (logits per head,
    probs per head, losses [CE light, CE booster, hint, sim_0, ...] or None without labels), from one fused call each
    way.  The caller checks rocket_head_usable first."""
    y = None if labels is None else labels.to(torch.float32).contiguous()
    flat = [t.contiguous() for h in heads for t in h]
    for light, booster in pairs:
        flat += [light.contiguous(), booster.detach().contiguous()]
    out = _RocketHead.apply((len(heads), len(pairs), float(eps), int(sim)), y, *flat)
    n = len(heads)
    losses = out[2 * n]
    return list(out[:n]), list(out[n:2 * n]), (list(losses.unbind(0)) if labels is not None else None)


def feature_based_sim(light: torch.Tensor, booster: torch.Tensor, sim: int) -> torch.Tensor:
    """rocket_launching.py:125-155 without sample weights: COSINE -0.1 mean_b <normalize(b), normalize(l)> with the
    booster detached; any other value the EUCLID branch sqrt(sum (b - l)^2) over the whole batch."""
    import torch.nn.functional as F

    b = booster.detach()
    if sim == ROCKET_COSINE:
        return -0.1 * torch.mean(torch.sum(torch.mul(F.normalize(b, p=2, dim=1), F.normalize(light, p=2, dim=1)), dim=1))
    return torch.sqrt(torch.sum(torch.square(b - light)))


def torch_rocket_head(heads, labels: Optional[torch.Tensor], eps: float = 0.0, pairs=(), sim: int = ROCKET_COSINE):
    """rocket_head in torch ops, as the reference computes it (the fallback on CPU tensors, under autocast, with TF32 on
    and outside the kernels' cover).  heads [(h, linear module)]."""
    logits = [lin(h) for h, lin in heads]
    probs = [torch.softmax(z, dim=1) for z in logits]
    return logits, probs, None if labels is None else torch_rocket_losses(logits, labels, eps, pairs, sim)


def torch_rocket_losses(logits: Sequence[torch.Tensor], labels: torch.Tensor, eps: float = 0.0, pairs=(),
                        sim: int = ROCKET_COSINE) -> List[Optional[torch.Tensor]]:
    """[CE light, CE booster, hint, sim_0, ...] of rocket_launching.py:182-245 from the heads' logits (light first;
    None where the booster head is absent): CrossEntropyLoss(mean, label_smoothing) on the label as a class index,
    MSELoss(mean)(logits_light, logits_booster.detach()) and feature_based_sim per pair."""
    import torch.nn.functional as F

    target = labels.to(torch.int64)
    ce = [F.cross_entropy(z, target, reduction="mean", label_smoothing=eps) for z in logits]
    losses = [ce[0], ce[1] if len(ce) > 1 else None,
              F.mse_loss(logits[0], logits[1].detach()) if len(logits) > 1 else None]
    losses += [feature_based_sim(light, booster, sim) for light, booster in pairs]
    return losses


# --------------------------------------------------------------------------------------------------------
# TDM multi-window DIN attention (tzrec/modules/sequence.py MultiWindowDINEncoder; csrc/tzk_tdm.cuh)
# --------------------------------------------------------------------------------------------------------
TDM_MAX_C = 128               # csrc/tzk_tdm.cuh: sequence width, a multiple of 4
TDM_MAX_HIDDEN = 64           # units of one attention layer (two per lane)
TDM_MAX_LAYERS = 3
TDM_MAX_WINDOWS = 32
TDM_MAX_SPAN = 256            # sum of the window lengths


def _attn_layers(mlp):
    """[(linear, activation)] of an attention MLP whose every Perceptron is exactly Linear(bias) + ReLU / one-slope
    PReLU, with one activation kind throughout; else None."""
    out = []
    for p in mlp.mlp:
        seq = p.perceptron
        if len(seq) != 2 or seq[0].bias is None:
            return None
        act = seq[1]
        if not (type(act) is torch.nn.ReLU or (type(act) is torch.nn.PReLU and act.weight.numel() == 1)):
            return None
        out.append((seq[0], act))
    if not out or len({type(a) for _, a in out}) != 1:
        return None
    return out


def multiwindow_din_usable(query: torch.Tensor, seq: torch.Tensor, mlp, windows: Sequence[int]) -> bool:
    """True when tzk_tdm_fwd / _bwd cover the encoder: fp32 query and rows, autocast and TF32 off, 4 <= C <= 128 with
    C % 4 == 0, Dq <= C, 1..3 attention layers of at most 64 units with bias and ReLU or one-slope PReLU (no BN, LN or
    dropout), 1..32 windows of total length <= 256, shared memory within the H100's 227 KB; on CUDA (on the CPU only a
    test backend that implements the kernels)."""
    if autocast_dtype(seq) is not None or query.dtype != torch.float32 or seq.dtype != torch.float32:
        return False
    C, Dq = seq.shape[1], query.shape[1]
    if not (4 <= C <= TDM_MAX_C and C % 4 == 0 and Dq <= C):
        return False
    layers = _attn_layers(mlp)
    if layers is None or len(layers) > TDM_MAX_LAYERS or any(l.out_features > TDM_MAX_HIDDEN for l, _ in layers):
        return False
    if not 1 <= len(windows) <= TDM_MAX_WINDOWS or min(windows) < 1 or sum(windows) > TDM_MAX_SPAN:
        return False
    if seq.is_cuda:
        if _backend is not None or torch.backends.cuda.matmul.allow_tf32:
            return False
        from ._lib import TDM_PRELU, TDM_RELU, TzkTdmArgs, lib

        a = TzkTdmArgs()
        a.C, a.Dq, a.L, a.n_layers = C, Dq, len(windows), len(layers)
        a.act = TDM_PRELU if type(layers[0][1]) is torch.nn.PReLU else TDM_RELU
        for w, n in enumerate(windows):
            a.windows[w] = int(n)
        for l, (lin, _) in enumerate(layers):
            a.hidden[l] = lin.out_features
        return lib().tzk_tdm_smem_bytes(ctypes.byref(a), 1) > 0
    return _backend is not None and hasattr(_backend, "tdm_fwd")


class _MultiWindowDin(torch.autograd.Function):
    """MultiWindowDINEncoder's attention, pooling and query block in one tzk_tdm_fwd call; every gradient in one
    tzk_tdm_bwd call.  params: per layer w, b (and the slope with PReLU), then lin_w, lin_b, act_w."""

    @staticmethod
    def forward(ctx, spec, query, seq, offsets, *params):
        windows, prelu, n_layers = spec
        layers, lin = _tdm_unflatten(params, prelu, n_layers)
        out, z = backend().tdm_fwd(query, seq, offsets, layers, *lin, windows, prelu)
        ctx.save_for_backward(query, seq, offsets, z, *params)
        ctx.spec = spec
        return out

    @staticmethod
    def backward(ctx, d_out):
        windows, prelu, n_layers = ctx.spec
        query, seq, offsets, z, *params = ctx.saved_tensors
        layers, lin = _tdm_unflatten(params, prelu, n_layers)
        d_q, d_seq, grads, d_lw, d_lb, d_aw = backend().tdm_bwd(query, seq, offsets, layers, *lin, windows, prelu, z,
                                                                d_out.contiguous())
        out = [None, d_q, d_seq, None]
        for dw, db, ds in grads:
            out += [dw, db] + ([ds] if prelu else [])
        return tuple(out + [d_lw, d_lb, d_aw])


def _tdm_unflatten(params, prelu: bool, n_layers: int):
    per = 3 if prelu else 2
    layers = [(params[per * l], params[per * l + 1], params[per * l + 2] if prelu else None) for l in range(n_layers)]
    return layers, params[per * n_layers:]


def multiwindow_din(query: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor, mlp, linear, active,
                    windows: Sequence[int]) -> torch.Tensor:
    """[B, (L + 1) C] of MultiWindowDINEncoder over jagged rows seq [N, C] (sample b: rows offsets[b] ..
    offsets[b + 1]) from one fused call each way.  The caller checks multiwindow_din_usable first."""
    layers = _attn_layers(mlp)
    prelu = type(layers[0][1]) is torch.nn.PReLU
    flat = []
    for lin, act in layers:
        flat += [lin.weight, lin.bias] + ([act.weight] if prelu else [])
    flat += [linear.weight, linear.bias, active.weight]
    return _MultiWindowDin.apply((tuple(int(w) for w in windows), prelu, len(layers)), query.contiguous(),
                                 seq.contiguous(), offsets, *[t.contiguous() for t in flat])


def torch_multiwindow_din(query: torch.Tensor, seq: torch.Tensor, offsets: torch.Tensor, mlp, linear, active,
                          windows: Sequence[int]) -> torch.Tensor:
    """multiwindow_din in torch ops over the same jagged rows (library GEMMs; the path under autocast, on CPU tensors
    and outside the kernels' cover).  The reference's padded rows give exact zeros and its rows past S are cropped, so
    over the real rows this is the reference up to the order of the sums."""
    N, C = seq.shape
    B = offsets.numel() - 1
    L, S = len(windows), int(sum(windows))
    seg = _segments(offsets, N)
    pos = torch.arange(N, device=seq.device) - offsets[:-1][seg]
    q = torch.nn.functional.pad(query, (0, C - query.shape[1])) if query.shape[1] < C else query
    qr = q[seg]
    a = active(linear(mlp(torch.cat([seq, qr * seq, qr], dim=-1))))           # [N, 1]
    keep = pos < S
    win_of = torch.repeat_interleave(torch.arange(L, device=seq.device),
                                     torch.tensor(list(windows), device=seq.device), output_size=S)
    idx = seg * L + win_of[pos.clamp(max=S - 1)]
    att = a * keep.unsqueeze(1) * seq
    pooled = torch.zeros((B * L, C), dtype=att.dtype, device=seq.device).index_add(0, idx, att)
    w = torch.tensor(list(windows), device=seq.device)
    cum = torch.cumsum(w, 0) - w
    lens = offsets[1:] - offsets[:-1]
    cnt = torch.clamp(torch.minimum(lens.unsqueeze(1) - cum.unsqueeze(0), w.unsqueeze(0)), min=1)
    res = pooled.view(B, L, C) / cnt.unsqueeze(2)
    return torch.cat([res, q.unsqueeze(1).to(res.dtype)], dim=1).reshape(B, -1)


# --------------------------------------------------------------------------------------------------------
# DCN-v2 low-rank cross network (tzrec/modules/interaction.py CrossV2; csrc/tzk_dcn_v2.cuh)
# --------------------------------------------------------------------------------------------------------
DCN_V2_MAX_D = 512            # csrc/tzk_dcn_v2.cuh: input width
DCN_V2_MAX_RANK = 64
DCN_V2_MAX_LAYERS = 8
# The model takes the fused path up to D r = 8192 (256 x 32, 128 x 64, 33 x 64).  The kernels accept up to 512 x 64,
# but on an H100 at B = 65536 the torch loop's library GEMMs beat them at D 256, L 3, r 64 (DESIGN.md §8), so wider
# products stay on the torch path.
DCN_V2_MAX_DR = 8192


def cross_v2_usable(x: torch.Tensor, u_kernels, v_kernels) -> bool:
    """True when tzk_dcn_v2_fwd / _bwd_data / _bwd_weight cover the cross network: fp32 input and weights, autocast and
    TF32 off, 1 <= D <= 512, 1 <= L <= 8, 1 <= r <= 64 with D r <= DCN_V2_MAX_DR, every v kernel with its bias, shared
    memory within the H100's 227 KB; on CUDA (on the CPU only a test backend that implements the kernels)."""
    if autocast_dtype(x) is not None or x.dtype != torch.float32 or x.dim() != 2:
        return False
    L = len(u_kernels)
    if not 1 <= L <= DCN_V2_MAX_LAYERS or len(v_kernels) != L:
        return False
    D, r = x.shape[1], u_kernels[0].out_features
    if not (1 <= D <= DCN_V2_MAX_D and 1 <= r <= DCN_V2_MAX_RANK and D * r <= DCN_V2_MAX_DR):
        return False
    for u, v in zip(u_kernels, v_kernels):
        if u.weight.dtype != torch.float32 or v.weight.dtype != torch.float32 or v.bias is None:
            return False
        if tuple(u.weight.shape) != (r, D) or tuple(v.weight.shape) != (D, r):
            return False
    if x.is_cuda:
        if _backend is not None or torch.backends.cuda.matmul.allow_tf32:
            return False
        from ._lib import TzkDcnV2Args, lib

        a = TzkDcnV2Args()
        a.D, a.L, a.r = D, L, r
        return all(lib().tzk_dcn_v2_smem_bytes(ctypes.byref(a), p) > 0 for p in range(3))
    return _backend is not None and hasattr(_backend, "dcn_v2_fwd")


class _CrossV2(torch.autograd.Function):
    """The whole cross network in one tzk_dcn_v2_fwd call; dx0 and every weight gradient from tzk_dcn_v2_bwd_data and
    tzk_dcn_v2_bwd_weight.  Saves x0, the weights and v [B, L r] only."""

    @staticmethod
    def forward(ctx, x0, wu, wv, bias):
        y, v = backend().dcn_v2_fwd(x0, wu, wv, bias)
        ctx.save_for_backward(x0, wu, wv, bias, v)
        return y

    @staticmethod
    def backward(ctx, dy):
        x0, wu, wv, bias, v = ctx.saved_tensors
        return backend().dcn_v2_bwd(x0, wu, wv, bias, v, dy.contiguous())


def cross_v2(x: torch.Tensor, u_kernels, v_kernels) -> torch.Tensor:
    """x_L of CrossV2 from one fused call each way.  The caller checks cross_v2_usable first."""
    wu = torch.stack([u.weight for u in u_kernels])
    wv = torch.stack([v.weight for v in v_kernels])
    bias = torch.stack([v.bias for v in v_kernels])
    return _CrossV2.apply(x.contiguous(), wu, wv, bias)


def torch_cross_v2(x: torch.Tensor, u_kernels, v_kernels) -> torch.Tensor:
    """CrossV2.forward of the reference in torch ops (the path on CPU tensors, under autocast, with TF32 on and outside
    the kernels' cover)."""
    x_l = x
    for u, v in zip(u_kernels, v_kernels):
        x_l = x * v(u(x_l)) + x_l
    return x_l


# --------------------------------------------------------------------------------------------------------
# sequence encoders of DEEP groups (tzrec/modules/sequence.py SelfAttentionEncoder / PoolingEncoder;
# csrc/tzk_seq_attn.cuh)
# --------------------------------------------------------------------------------------------------------
SELF_ATTN_MAX_HD = 128        # csrc/tzk_seq_attn.cuh: head width


def self_attn_pool_usable(q: torch.Tensor, H: int, dropout: float, training: bool) -> bool:
    """True when tzk_self_attn_pool_fwd / _bwd cover the attention: fp32 rows, autocast off, 1 <= hd <= 128, no dropout
    in training (torch's dropout RNG cannot be matched); on CUDA (on the CPU only a test backend that implements the
    kernels)."""
    if autocast_dtype(q) is not None or q.dtype != torch.float32 or q.dim() != 2 or H < 1 or q.shape[1] % H != 0:
        return False
    if not 1 <= q.shape[1] // H <= SELF_ATTN_MAX_HD or (dropout > 0.0 and training):
        return False
    if q.is_cuda:
        return _backend is None
    return _backend is not None and hasattr(_backend, "self_attn_pool_fwd")


class _SelfAttnPool(torch.autograd.Function):
    """The attention core in one tzk_self_attn_pool_fwd call (saves the lse [N, H] only); dq, dk, dv in one
    tzk_self_attn_pool_bwd call."""

    @staticmethod
    def forward(ctx, q, k, v, offsets, H, max_len):
        pooled, lse = backend().self_attn_pool_fwd(q, k, v, offsets, H, max_len)
        ctx.save_for_backward(q, k, v, offsets, lse)
        ctx.spec = (H, max_len)
        return pooled

    @staticmethod
    def backward(ctx, d_pooled):
        q, k, v, offsets, lse = ctx.saved_tensors
        dq, dk, dv = backend().self_attn_pool_bwd(q, k, v, offsets, *ctx.spec, lse, d_pooled.contiguous())
        return dq, dk, dv, None, None, None


def self_attn_pool(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, offsets: torch.Tensor, H: int,
                   max_len: int = 0) -> torch.Tensor:
    """pooled [B, E]: per sample b and head, sum_i sum_j p_ij v_j over the first L_b = min(len_b, max_len) rows (0:
    all) of the in-projected jagged rows q, k, v [N, E], p = softmax_j((q_i sqrt(1/hd)) . k_j).  One fused call each
    way; the caller checks self_attn_pool_usable first."""
    return _SelfAttnPool.apply(q.contiguous(), k.contiguous(), v.contiguous(), offsets, int(H), int(max_len))


def torch_self_attn_pool(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, offsets: torch.Tensor, H: int,
                         max_len: int = 0, dropout: float = 0.0, training: bool = False) -> torch.Tensor:
    """self_attn_pool in torch ops (the path under autocast, on CPU tensors, with dropout in training and outside the
    kernels' cover): the kept rows padded to the batch's longest kept length (one host read), every key beyond a
    sample's length masked, and every padded query row's probabilities zeroed after the softmax, so no row is NaN and
    every gradient is finite.  `dropout` applies to the attention probabilities, as in nn.MultiheadAttention."""
    N, E = q.shape
    B, hd = offsets.numel() - 1, E // H
    lens = offsets[1:] - offsets[:-1]
    kept = torch.clamp_max(lens, max_len) if max_len > 0 else lens
    T = int(kept.max()) if B > 0 else 0
    seg = _segments(offsets, N)
    pos = torch.arange(N, device=q.device) - offsets[:-1][seg]
    keep = pos < kept[seg]
    idx = seg[keep] * max(T, 1) + pos[keep]

    def pad(x):
        out = torch.zeros((B * max(T, 1), E), dtype=x.dtype, device=x.device).index_copy(0, idx, x[keep])
        return out.view(B, max(T, 1), H, hd).transpose(1, 2)                    # [B, H, T, hd]

    qp, kp, vp = pad(q) * math.sqrt(1.0 / hd), pad(k), pad(v)
    valid = torch.arange(max(T, 1), device=q.device).unsqueeze(0) < kept.unsqueeze(1)          # [B, T]
    s = torch.matmul(qp, kp.transpose(-1, -2)).masked_fill(~valid[:, None, None, :], torch.finfo(qp.dtype).min)
    p = torch.softmax(s, dim=-1) * valid[:, None, :, None].to(qp.dtype)
    if dropout > 0.0 and training:
        p = torch.nn.functional.dropout(p, dropout, True)
    c = p.sum(dim=-2)                                                           # [B, H, T]
    return torch.matmul(c.unsqueeze(-2), vp).reshape(B, E)


def jagged_pool_usable(seq: torch.Tensor) -> bool:
    """True when tzk_jagged_pool_fwd / _bwd take the pooling: fp32 rows, autocast off; on CUDA (on the CPU only a test
    backend that implements the kernels)."""
    if autocast_dtype(seq) is not None or seq.dtype != torch.float32 or seq.dim() != 2:
        return False
    if seq.is_cuda:
        return _backend is None
    return _backend is not None and hasattr(_backend, "jagged_pool_fwd")


class _JaggedPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seq, offsets, max_len, mean):
        ctx.save_for_backward(offsets)
        ctx.spec = (seq.shape[0], max_len, mean)
        return backend().jagged_pool_fwd(seq, offsets, max_len, mean)

    @staticmethod
    def backward(ctx, d_out):
        offsets, = ctx.saved_tensors
        N, max_len, mean = ctx.spec
        return backend().jagged_pool_bwd(d_out.contiguous(), offsets, N, max_len, mean), None, None, None


def jagged_pool(seq: torch.Tensor, offsets: torch.Tensor, max_len: int = 0, mean: bool = True) -> torch.Tensor:
    """[B, D]: the sum, or the mean over max(L_b, 1), of each sample's first L_b = min(len_b, max_len) rows (0: all)
    of jagged rows seq [N, D], one fused call each way.  The caller checks jagged_pool_usable first."""
    return _JaggedPool.apply(seq.contiguous(), offsets, int(max_len), bool(mean))


def torch_jagged_pool(seq: torch.Tensor, offsets: torch.Tensor, max_len: int = 0, mean: bool = True) -> torch.Tensor:
    """jagged_pool in torch ops over the same rows (index_add into the samples; no host read)."""
    N, B = seq.shape[0], offsets.numel() - 1
    seg = _segments(offsets, N)
    lens = offsets[1:] - offsets[:-1]
    rows = seq
    if max_len > 0:
        pos = torch.arange(N, device=seq.device) - offsets[:-1][seg]
        rows = seq * (pos < max_len).unsqueeze(1).to(seq.dtype)
        lens = torch.clamp_max(lens, max_len)
    out = torch.zeros((B, seq.shape[1]), dtype=seq.dtype, device=seq.device).index_add(0, seg, rows)
    return out / torch.clamp_min(lens, 1).unsqueeze(1).to(out.dtype) if mean else out
