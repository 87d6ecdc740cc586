"""Reference of weighted id features: per-sample weights in the pooled lookup and in the fused sparse update.

TEST INFRASTRUCTURE.  A numpy restatement of what csrc/tzk_gather.cu (pooled_gather_fwd_weighted_kernel) and
csrc/tzk_bwd.cu (fused_apply_weighted_kernel) compute, which restate fbgemm_gpu's weighted TBE ([EXT], unverified
against a real wheel: DESIGN.md §5) as torchrec's sharded lookup drives it with `features.weights_or_none()`:

  forward   out[b, col_f : +D] = sum_{l in bag(f,b)} w[l] * row(ids[l]) in list order, fp32 (fused multiply-add), MEAN / L
  backward  position l contributes grad_scale * w[l] * grad_out[b, col_f : +D] (/ L for MEAN) to its row; the
            contributions of a row are added in the stable (table, row) order, then the optimizer applies its update

`WeightedOracleKernels` is tests/sparse_optim_ref.ExtOracleKernels with the weights added: the update is the existing
un-pooled (per-position) update over gradient rows that already carry grad_scale * w[l] (/ L), so every optimizer kind
of the oracles serves weighted bags unchanged.  The C oracle has no weighted lookup: with use_c it raises.
"""
import numpy as np
import torch

from oracle import tzk_oracle as O
from oracle_backend import _np, _tables
from sparse_optim_ref import ExtOracleKernels

from torcheasyrec_b200.kernels import FeatureLayout

f32 = np.float32


def fma32(w, r, acc):
    """fp32 fmaf(w, r, acc): the product of two fp32 values is exact in float64, the sum is rounded once there and once
    to fp32 (exact for the dyadic test data; within an ulp otherwise)."""
    return (w.astype(np.float64) * r.astype(np.float64) + acc.astype(np.float64)).astype(f32)


def pooled_lookup_weighted(tables, feat_table, feat_pool, ids, offsets, B, psw):
    """Weighted pooled lookup, in list order: acc = w[l0] * row(l0), then acc = fmaf(w[l], row(l), acc)."""
    F = len(feat_table)
    dims = [tables[t].shape[1] for t in feat_table]
    out = np.zeros((B, int(sum(dims))), dtype=f32)
    col = 0
    for f in range(F):
        W = tables[feat_table[f]]
        D = W.shape[1]
        for b in range(B):
            s, e = int(offsets[f * B + b]), int(offsets[f * B + b + 1])
            if e == s:
                continue
            fid = O._clamp_ids(ids[s:e], W.shape[0])
            acc = (f32(psw[s]) * W[fid[0]]).astype(f32)
            for j in range(1, e - s):
                acc = fma32(np.full(D, psw[s + j], f32), W[fid[j]], acc)
            if feat_pool[f] == O.POOL_MEAN:
                acc = (acc * (f32(1.0) / f32(e - s))).astype(f32)
            out[b, col:col + D] = acc
        col += D
    return out


def position_grads(grad_out, lay, offsets, B, psw, grad_scale):
    """One gradient row per id position, as the kernel forms it: g[bag] * (grad_scale (/ L)) * w[l], all fp32."""
    nnz = int(offsets[-1])
    rows = np.zeros((nnz, lay.max_dim), dtype=f32)
    gs = f32(grad_scale)
    for f in range(lay.num_features):
        D, c = lay.dim[f], lay.col[f]
        for b in range(B):
            s, e = int(offsets[f * B + b]), int(offsets[f * B + b + 1])
            if e == s:
                continue
            sc = gs / f32(e - s) if lay.pool[f] == O.POOL_MEAN else gs
            for l in range(s, e):
                rows[l, :D] = grad_out[b, c:c + D].astype(f32) * f32(sc * f32(psw[l]))
    return rows


class WeightedOracleKernels(ExtOracleKernels):
    """Test backend that knows weighted bags; unweighted calls go to the oracles unchanged."""

    def _no_c(self):
        if self.use_c:
            raise NotImplementedError("the C oracle has no weighted lookup: use the numpy oracle for weighted id features")

    def pooled_gather_fwd(self, weights, lay, ids, offsets, B, out=None, per_sample_weights=None):
        if per_sample_weights is None:
            return super().pooled_gather_fwd(weights, lay, ids, offsets, B, out)
        self._no_c()
        tabs, ft = _tables(weights, lay)
        res = torch.from_numpy(pooled_lookup_weighted(tabs, ft, lay.pool, _np(ids), _np(offsets), B,
                                                      _np(per_sample_weights)))
        if out is not None:
            out.copy_(res)
            return out
        return res

    def permute_weights(self, weights, in_offsets, out_offsets, perm, B, out_nnz):
        w, off, p = _np(weights), _np(in_offsets), _np(perm)
        parts = [w[off[k * B]:off[(k + 1) * B]] for k in p]
        return torch.from_numpy(np.concatenate(parts).astype(np.float32) if parts else w[:0])

    def fused_bwd(self, optimizer, pooled, grad_out, weights, state, lay, ids, offsets, B, lr, eps, grad_scale=1.0,
                  **ex):
        psw = ex.pop("per_sample_weights", None)
        if psw is None:
            return super().fused_bwd(optimizer, pooled, grad_out, weights, state, lay, ids, offsets, B, lr, eps,
                                     grad_scale, **ex)
        self._no_c()
        assert pooled, "per-sample weights are a pooled-lookup input"
        off, idn = _np(offsets), _np(ids)
        rows = position_grads(_np(grad_out), lay, off, B, _np(psw), grad_scale)
        # the per-position (un-pooled) update takes one dim per call: one call per dim, each with its features
        for D in sorted(set(lay.dim)):
            fs = [f for f in range(lay.num_features) if lay.dim[f] == D]
            seg = [(int(off[f * B]), int(off[(f + 1) * B])) for f in fs]
            sub_ids = np.concatenate([idn[s:e] for s, e in seg]) if seg else idn[:0]
            sub_g = np.concatenate([rows[s:e, :D] for s, e in seg], axis=0)
            bounds = np.concatenate([[0], np.cumsum([e - s for s, e in seg])]).astype(np.int64)
            sub = FeatureLayout(w_off=[lay.w_off[f] for f in fs], rows=[lay.rows[f] for f in fs], dim=[D] * len(fs),
                                col=[0] * len(fs), pool=[O.POOL_SUM] * len(fs), key_base=[lay.key_base[f] for f in fs],
                                total_keys=lay.total_keys, total_dim=D, arena_elems=lay.arena_elems,
                                stride=None if lay.stride is None else [lay.stride[f] for f in fs],
                                interleaved=lay.interleaved)
            super().fused_bwd(optimizer, False, torch.from_numpy(np.ascontiguousarray(sub_g)), weights, state, sub,
                              torch.from_numpy(sub_ids.astype(np.int64)), torch.from_numpy(bounds), 1, lr, eps, 1.0,
                              **ex)
