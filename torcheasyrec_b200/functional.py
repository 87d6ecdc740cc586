"""Autograd-aware operators of the hot path, each a thin shell over one or two tzk kernels.

The compute backend is `CudaKernels` (kernels.py).  `use_backend()` exists so that the host-side logic
(sharding plans, all-to-all plumbing, regroup plans) can be unit-tested on a CPU box by *tests* that inject
their own checker backend; the package itself never provides one and every default path raises on CPU
tensors.
"""

import contextlib
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


def dot_interaction(features: torch.Tensor) -> torch.Tensor:
    """InteractionArch.forward (tzrec/modules/interaction.py:80-91): [B,N,D] -> [B, N(N-1)/2].

    Under autocast this is the reference's torch formulation: bmm is on autocast's lower-precision list."""
    if autocast_dtype(features) is not None:
        return _torch_dot_interaction(features)
    B, N, D = features.shape
    return _DotInteract.apply(None, features.reshape(B, N * D), N, D, False, False)


def dlrm_interaction(dense_feat: Optional[torch.Tensor], sparse_feat: torch.Tensor, num_sparse: int, dim: int,
                     with_dense: bool = True, with_sparse: bool = True, aligned: bool = False):
    """Fused DLRM.predict glue (tzrec/models/dlrm.py:113-131):
    cat([interaction(cat([dense[:,None,:], sparse.view(B,Ns,D)], 1)), dense, sparse], -1) in one pass.

    aligned=False -> the reference's exact column layout [P | dense | sparse].
    aligned=True  -> (tensor, in_map): zero columns are inserted after the P interaction terms and at the row end so
    that every block and every row starts on a 16-B boundary; `in_map` = [(src_col, dst_col, length), ...] tells the
    consuming Linear where the reference's columns live (dense_gemm.linear pads its weight accordingly).

    Under autocast this is the reference's torch formulation in the reference's layout (with aligned=True the map is
    None): autocast rounds the bmm to its dtype and the concatenations promote back to fp32, as in dlrm.py.  DLRM-Criteo
    under bf16 autocast has its own kernel (dense_gemm.InteractBf16Fn)."""
    if autocast_dtype(sparse_feat) is not None:
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
