"""Weighted id features on the peer-memory sparse step (peer_exchange.PeerState + csrc/tzk_peer.cu), without a GPU.

The per-sample weights never leave the sample's rank: its gather pools w[l] * row, its bucketize records every wire
slot's weight in a local buffer and its push sends w * g (/ L); the owner's update is the unweighted one with the 1/W
gradient scale.  W ranks run as threads of this process (tests/test_peer_exchange_model.py's plumbing); the peer
kernels run as a loop-level model ("model") or from csrc/tzk_peer.cu compiled for the host ("source").  Checked against
the unsharded weighted reference (tests/weighted_ref.py) on the key-major concatenation of the W local batches:
  * dyadic ids / gradients / weights / tables with W in {2, 4}: outputs and updated rows bit-exact;
  * otherwise within the sharded tolerances (outputs 1e-6, tables 5e-5);
  * all-ones weights: the unweighted peer step bit for bit (outputs, tables, optimizer state);
  * the pull transport and weights that require grad raise on the host."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import test_peer_exchange_model as M  # noqa: E402  (sets TZK_PEER_MIRROR_ROWS: some tables mirrored, some remote)
from oracle_backend import OracleKernels, _np  # noqa: E402
from weighted_ref import WeightedOracleKernels, fma32  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200 import peer_exchange  # noqa: E402
from torcheasyrec_b200.distributed import TABLE_WISE, _DimGroup, make_plan  # noqa: E402
from torcheasyrec_b200.embedding_modules import (EmbeddingBagCollection, SparseOptimizerSpec,  # noqa: E402
                                                 output_names_by_table)
from torcheasyrec_b200.kernels import OPT_ACCUM_OUT, OPT_ADAGRAD  # noqa: E402

P, I32, I64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
f32 = np.float32


@pytest.fixture(scope="module")
def host_peer_lib(tmp_path_factory):
    """csrc/tzk_peer.cu compiled for the host (tests/native/cuda_cpu_shim.h), weighted entry points bound too."""
    exp = os.path.join(HERE, "native")
    out = str(tmp_path_factory.mktemp("wshim") / "libtzk_peer_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", exp, "-x",
                    "c++", os.path.join(os.path.dirname(HERE), "torcheasyrec_b200", "csrc", "tzk_peer.cu"), "-shared",
                    "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    L.tzk_peer_pooled_gather_fwd.argtypes = [P, P, P, P, P, P, P, P, P, P, I32, I32, I32, I32, P, I64, P, P, P]
    L.tzk_peer_pooled_gather_fwd_sel.argtypes = [P, P, P, P, P, P, P, P, P, P, I32, I32, I32, I32, P, I64, P, P, P, I32, P]
    L.tzk_peer_pooled_gather_fwd_weighted.argtypes = [P, P, P, P, P, P, P, P, P, P, I32, I32, I32, I32, P, I64, P, P, P,
                                                      P, I32, P]
    L.tzk_peer_mirror_refresh.argtypes = [P, I32, P, P, P, P, I32, P, P]
    L.tzk_peer_bucketize_workspace_bytes.restype = ctypes.c_size_t
    L.tzk_peer_bucketize_workspace_bytes.argtypes = [I32, I32, I32]
    L.tzk_peer_bucketize.argtypes = [P, P, I32, I32, I32, P, P, P, P, I32, I64, P, P, P, P, ctypes.c_size_t, P]
    L.tzk_peer_bucketize_weighted.argtypes = [P, P, I32, I32, I32, P, P, P, P, I32, I64, P, P, P, P, ctypes.c_size_t,
                                              P, P, P]
    L.tzk_peer_publish_grad.argtypes = [P, I64, P, P, P, P, I32, I32, P, I64, P]
    L.tzk_peer_allreduce_mean.argtypes = [P, I32, I64, P, P]
    L.tzk_peer_push_grad.argtypes = [P, P, I64, P, P, P, P, P, I32, I32, I64, I32, I32, I32, P]
    L.tzk_peer_push_grad_weighted.argtypes = [P, P, I64, P, P, P, P, P, I32, I32, I64, I32, I32, I32, P, P]
    return L


class WeightedPeerModel(OracleKernels):
    """The peer kernels' loop-level model with weighted bags, plus the owner-side small-table ops (the sort remembers
    the weights; TZK_OPT_ACCUM_OUT forms every entry as the weighted run kernels do: ((grad_scale / L) * w) * g)."""

    def peer_pooled_gather_fwd(self, tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets, B, W,
                               out=None, mirror=None, feat_mirror_off=None, feat_sel=None, per_sample_weights=None):
        if per_sample_weights is None:
            return super().peer_pooled_gather_fwd(tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets,
                                                  B, W, out, mirror, feat_mirror_off, feat_sel)
        sel = None if feat_sel is None else set(feat_sel.tolist())
        if mirror is not None:
            self._check_mirror(tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, W, mirror, feat_mirror_off)
        F = lay.num_features
        blocks, owners, rows, w_off = feat_block.tolist(), feat_owner.tolist(), feat_rows.tolist(), rf_w_off.tolist()
        idl, off, w = ids.tolist(), offsets.tolist(), _np(per_sample_weights)
        o = out.numpy() if sel is not None else np.zeros((B, lay.total_dim), dtype=f32)
        for f in range(F):
            if sel is not None and f not in sel:
                continue
            D, col = lay.dim[f], lay.col[f]
            for b in range(B):
                s, e = off[f * B + b], off[f * B + b + 1]
                acc = np.zeros(D, dtype=f32)
                for l in range(s, e):
                    i = idl[l] if 0 <= idl[l] < rows[f] else 0
                    r, loc = self._owner_of(i, blocks[f], owners[f], W)
                    row = tables.everyone[r].numpy()[w_off[r * F + f] + loc * D:w_off[r * F + f] + (loc + 1) * D]
                    acc = (f32(w[l]) * row).astype(f32) if l == s else fma32(np.full(D, w[l], f32), row, acc)
                if lay.pool[f] == 1 and e > s:
                    acc = (acc * (f32(1.0) / f32(e - s))).astype(f32)
                o[b, col:col + D] = acc
        if sel is not None:
            return out
        res = torch.from_numpy(o)
        if out is not None:
            out.copy_(res)
            return out
        return res

    def peer_bucketize(self, ids, offsets, F, B, W, feat_block, feat_owner, feat_rows, rf_key_base, pooled, cap,
                       wire_key, wire_idx, counts, per_sample_weights=None, wire_w=None):
        super().peer_bucketize(ids, offsets, F, B, W, feat_block, feat_owner, feat_rows, rf_key_base, pooled, cap,
                               wire_key, wire_idx, counts)
        if per_sample_weights is None:
            return
        assert pooled and wire_w is not None
        blocks, owners, rows = feat_block.tolist(), feat_owner.tolist(), feat_rows.tolist()
        idl, off, w = ids.tolist(), offsets.tolist(), _np(per_sample_weights)
        fill = [0] * W
        for bag in range(F * B):        # the same slot order as the ids' (feature, bag, position)
            f = bag // B
            if blocks[f] <= 0:
                continue
            for l in range(off[bag], off[bag + 1]):
                i = idl[l] if 0 <= idl[l] < rows[f] else 0
                r, _ = self._owner_of(i, blocks[f], owners[f], W)
                if fill[r] < cap:
                    wire_w[r * cap + fill[r]] = float(w[l])
                fill[r] += 1

    def peer_push_grad(self, recv, grad, lay, offsets, wire_idx, counts, me, W, cap, B, pooled, wire_w=None):
        if wire_w is None:
            return super().peer_push_grad(recv, grad, lay, offsets, wire_idx, counts, me, W, cap, B, pooled)
        g, off, ww = _np(grad), _np(offsets), _np(wire_w)
        D = lay.dim[0]
        for r in range(W):
            dst = recv.everyone[r].numpy()
            for j in range(int(counts[r])):
                idx = int(wire_idx[r * cap + j])
                f, b = divmod(idx, B)
                sc = f32(1.0) / f32(off[idx + 1] - off[idx]) if lay.pool[f] == 1 else f32(1.0)
                sc = f32(sc * f32(ww[r * cap + j]))                 # (1/L) * w first, then the slice
                dst[(me * cap + j) * D:(me * cap + j + 1) * D] = g[b, lay.col[f]:lay.col[f] + D] * sc

    def fused_bwd_workspace_bytes(self, lay, nnz, weighted=False):
        return 256

    def fused_bwd_sort(self, pooled, lay, ids, offsets, B, ws, per_sample_weights=None):
        super().fused_bwd_sort(pooled, lay, ids, offsets, B, ws)
        if not hasattr(self, "_local_w"):
            self._local_w = {}
        self._local_w[ws.data_ptr()] = None if per_sample_weights is None else _np(per_sample_weights).copy()

    def fused_bwd_apply(self, optimizer, pooled, grad_out, weights, state, lay, offsets, nnz, B, lr, eps, grad_scale, ws,
                        **ex):
        psw = ex.pop("per_sample_weights", None)
        if optimizer != OPT_ACCUM_OUT or psw is None:
            return super().fused_bwd_apply(optimizer, pooled, grad_out, weights, state, lay, offsets, nnz, B, lr, eps,
                                           grad_scale, ws, **ex)
        assert pooled and self._local_w[ws.data_ptr()] is not None
        ids, off, B, _ = self._local_sorted[ws.data_ptr()]
        w = self._local_w[ws.data_ptr()]
        g = _np(grad_out)
        Pm, Fl = weights.numpy(), state.numpy()
        sums = {}
        for f in range(lay.num_features):
            if lay.rows[f] <= 0:
                continue
            D = lay.dim[f]
            for bag in range(f * B, (f + 1) * B):
                L = off[bag + 1] - off[bag]
                for l in range(off[bag], off[bag + 1]):
                    i = ids[l] if 0 <= ids[l] < lay.rows[f] else 0
                    sc = f32(grad_scale) / f32(L) if lay.pool[f] == 1 else f32(grad_scale)
                    sc = f32(sc * f32(w[l]))
                    row = g[bag - f * B, lay.col[f]:lay.col[f] + D].astype(f32) * sc
                    key = lay.key_base[f] + i
                    cur = sums.get(key)
                    sums[key] = (row if cur is None else cur[0] + row, lay.w_off[f] + i * D, D)
        for key, (acc, o, D) in sums.items():
            Pm[o:o + D] = acc
            Fl[key] = 1


class WeightedPeerSource(WeightedPeerModel, M.SourceKernels):
    """The weighted peer kernels executed from csrc/tzk_peer.cu's host-compiled source; owner side as the model."""

    name = "oracle+weighted-peer-source"

    def peer_pooled_gather_fwd(self, tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets, B, W,
                               out=None, mirror=None, feat_mirror_off=None, feat_sel=None, per_sample_weights=None):
        if per_sample_weights is None:
            return M.SourceKernels.peer_pooled_gather_fwd(self, tables, rf_w_off, feat_rows, feat_block, feat_owner, lay,
                                                          ids, offsets, B, W, out, mirror, feat_mirror_off, feat_sel)
        dim, col, pool = self._lay(lay)
        out = torch.full((B, lay.total_dim), float("nan")) if out is None else out
        rc = self.L.tzk_peer_pooled_gather_fwd_weighted(
            tables.ptrs, rf_w_off.data_ptr(), feat_rows.data_ptr(), feat_block.data_ptr(), feat_owner.data_ptr(),
            dim.data_ptr(), col.data_ptr(), pool.data_ptr(), ids.data_ptr(), offsets.data_ptr(), lay.num_features, B, W,
            (lay.max_dim + 3) // 4 * 4, out.data_ptr(), lay.total_dim, None if mirror is None else mirror.data_ptr(),
            None if feat_mirror_off is None else feat_mirror_off.data_ptr(), per_sample_weights.data_ptr(),
            None if feat_sel is None else feat_sel.data_ptr(), 0 if feat_sel is None else feat_sel.numel(), None)
        assert rc == 0, rc
        return out

    def peer_bucketize(self, ids, offsets, F, B, W, feat_block, feat_owner, feat_rows, rf_key_base, pooled, cap,
                       wire_key, wire_idx, counts, per_sample_weights=None, wire_w=None):
        if per_sample_weights is None:
            return M.SourceKernels.peer_bucketize(self, ids, offsets, F, B, W, feat_block, feat_owner, feat_rows,
                                                  rf_key_base, pooled, cap, wire_key, wire_idx, counts)
        nb = self.L.tzk_peer_bucketize_workspace_bytes(F, B, W)
        ws = torch.zeros(nb // 4 + 1, dtype=torch.int32)
        rc = self.L.tzk_peer_bucketize_weighted(ids.data_ptr(), offsets.data_ptr(), F, B, W, feat_block.data_ptr(),
                                                feat_owner.data_ptr(), feat_rows.data_ptr(), rf_key_base.data_ptr(),
                                                int(pooled), cap, wire_key.data_ptr(), wire_idx.data_ptr(),
                                                counts.data_ptr(), ws.data_ptr(), nb, per_sample_weights.data_ptr(),
                                                wire_w.data_ptr(), None)
        assert rc == 0, rc

    def peer_push_grad(self, recv, grad, lay, offsets, wire_idx, counts, me, W, cap, B, pooled, wire_w=None):
        if wire_w is None:
            return M.SourceKernels.peer_push_grad(self, recv, grad, lay, offsets, wire_idx, counts, me, W, cap, B, pooled)
        _, col, pool = self._lay(lay)
        grad = grad.contiguous()
        rc = self.L.tzk_peer_push_grad_weighted(recv.ptrs, grad.data_ptr(), grad.shape[1], col.data_ptr(),
                                                pool.data_ptr(), offsets.data_ptr(), wire_idx.data_ptr(),
                                                counts.data_ptr(), me, W, cap, B, lay.dim[0], int(pooled),
                                                wire_w.data_ptr(), None)
        assert rc == 0, rc


def _bags(rng, F, B, feat_rows, dyadic):
    """Ragged bags with empty ones.  Dyadic data: lengths in {0, 1, 2, 4}, so a MEAN bag's 1/L is exact too."""
    lens = rng.choice([0, 1, 2, 4], F * B) if dyadic else rng.integers(0, 5, F * B)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = np.concatenate([rng.integers(0, feat_rows[b // B], lens[b]) for b in range(F * B)] + [np.zeros(0, np.int64)])
    return torch.from_numpy(ids.astype(np.int64)), torch.from_numpy(off)


def _weights(rng, n, dyadic):
    """Per-sample weights with negative ones (dyadic: k/4, |k| <= 8, zero included)."""
    w = rng.integers(-8, 9, n) / 4.0 if dyadic else rng.standard_normal(n) * 1.5
    return torch.from_numpy(w.astype(f32))


def _run_peer(cfgs, plan, W, B, spec, full, batches, weights, grads, backend, tag, steps=2):
    """W ranks as threads: `steps` peer steps (gather -> prep -> backward) on the sharded twin of `full`.
    Returns (groups, outs[step][rank])."""
    names = output_names_by_table(cfgs)
    groups = []
    for r in range(W):
        g = _DimGroup(cfgs, plan, r, W, torch.device("cpu"), True, names)
        g.static_alpha = 2.5
        g.local.set_optimizer(spec)
        for t, c in enumerate(cfgs):
            n = g.local._table_rows[t]
            if n:
                start = 0 if plan[c.name].kind == TABLE_WISE else r * plan[c.name].block
                g.local.set_table_weight(t, full.table_weight(t)[start:start + n])
        groups.append(g)
    F = groups[0].F
    registry, outs = {}, [[None] * W for _ in range(steps)]
    budget = [B * 4] * F

    def body(r, tbar):
        class St(M._sim_mixin(registry, tbar, tag), peer_exchange.PeerState):
            pass

        st = St(groups[r], plan, None, B, budget)
        ids, offs = batches[r]
        psw = None if weights is None else weights[r]
        for s in range(steps):
            outs[s][r] = st.gather(ids, offs, psw)
            st.prep(ids, offs, psw)
            st.backward(grads[r], offs)

    with Fn.use_backend(backend):
        M._run_ranks(W, body)
    assert all(int(g.overflow.item()) == 0 for g in groups)
    return groups, outs


def _gathered(groups, plan, cfgs, full, t):
    sh = plan[cfgs[t].name]
    got = torch.zeros_like(full.table_weight(t))
    for r, g in enumerate(groups):
        n = g.local._table_rows[t]
        if n:
            start = 0 if sh.kind == TABLE_WISE else r * sh.block
            got[start:start + n] = g.local.table_weight(t)
    return got


def _setup(W, dyadic, seed):
    rng = np.random.default_rng(seed)
    cfgs = M._pooled_configs()             # SUM and MEAN tables, one shared table, a 2-row table, a table-wise one
    B, D = 12, 16
    plan = make_plan(cfgs, W, "row_wise", {"t_tw": [TABLE_WISE], "t_tiny": [TABLE_WISE]})
    spec = SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.05)
    with Fn.use_backend(OracleKernels()):
        full = EmbeddingBagCollection(cfgs, device="cpu")
        full.set_optimizer(spec)
    if dyadic:
        full.weights.data.copy_(torch.from_numpy((rng.integers(-16, 17, full.weights.numel()) / 16.0).astype(f32)))
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows, dyadic) for _ in range(W)]
    weights = [_weights(rng, b[0].numel(), dyadic) for b in batches]
    if dyadic:
        grads = [torch.from_numpy((rng.integers(-8, 9, (B, F * D)) / 8.0).astype(f32)) for _ in range(W)]
    else:
        grads = [torch.from_numpy(rng.standard_normal((B, F * D)).astype(f32)) for _ in range(W)]
    return cfgs, plan, spec, full, F, B, batches, weights, grads


@pytest.mark.parametrize("kernels", ["model", "source"])
@pytest.mark.parametrize("small_bwd", ["1", "0"])
@pytest.mark.parametrize("W,dyadic", [(2, True), (4, True), (3, False), (4, False)])
def test_weighted_peer_step_matches_unsharded(W, dyadic, small_bwd, kernels, host_peer_lib, monkeypatch):
    """Two weighted peer steps against the unsharded weighted reference on the concatenated batch (grad / W)."""
    monkeypatch.setenv("TZK_PEER_SMALL_BWD", small_bwd)
    cfgs, plan, spec, full, F, B, batches, weights, grads = _setup(W, dyadic, 40 + W + 10 * dyadic)
    backend = WeightedPeerModel() if kernels == "model" else WeightedPeerSource(host_peer_lib)
    groups, outs = _run_peer(cfgs, plan, W, B, spec, full, batches, weights, grads, backend, "w")

    ref = WeightedOracleKernels()
    ids, offs = [b[0] for b in batches], [b[1] for b in batches]
    cat_ids, cat_off = M._cat_key_major(ids, offs, F, B, W)
    cat_w = torch.cat([weights[r][offs[r][f * B]:offs[r][(f + 1) * B]] for f in range(F) for r in range(W)])
    cat_grad = torch.cat(grads) / W
    for step in range(2):
        for r in range(W):
            want = ref.pooled_gather_fwd(full.weights.data, full.layout, ids[r], offs[r], B,
                                         per_sample_weights=weights[r])
            if dyadic or step == 0:
                np.testing.assert_array_equal(outs[step][r].numpy(), want.numpy(), err_msg=f"step {step} rank {r}")
            else:
                np.testing.assert_allclose(outs[step][r].numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
        ref.fused_bwd(spec.kind, True, cat_grad, full.weights.data, full.opt_state, full.layout, cat_ids, cat_off,
                      B * W, spec.lr, spec.eps, 1.0, per_sample_weights=cat_w)
    for t, c in enumerate(cfgs):
        got = _gathered(groups, plan, cfgs, full, t)
        if dyadic:
            np.testing.assert_array_equal(got.numpy(), full.table_weight(t).numpy(), err_msg=c.name)
        else:
            np.testing.assert_allclose(got.numpy(), full.table_weight(t).numpy(), rtol=5e-5, atol=1e-6, err_msg=c.name)


@pytest.mark.parametrize("kernels", ["model", "source"])
def test_all_ones_weights_are_the_unweighted_peer_step(kernels, host_peer_lib):
    """Weights of 1: the weighted gather, bucketize and push, and the weighted small-table sums, give every bit of
    the unweighted peer step — outputs, tables and the Adagrad state."""
    W = 3
    cfgs, plan, spec, full, F, B, batches, _, grads = _setup(W, False, 77)
    ones = [torch.ones(b[0].numel()) for b in batches]
    mk = (lambda: WeightedPeerModel()) if kernels == "model" else (lambda: WeightedPeerSource(host_peer_lib))
    g_w, o_w = _run_peer(cfgs, plan, W, B, spec, full, batches, ones, grads, mk(), "ones")
    g_u, o_u = _run_peer(cfgs, plan, W, B, spec, full, batches, None, grads, mk(), "plain")
    for step in range(2):
        for r in range(W):
            np.testing.assert_array_equal(o_w[step][r].numpy(), o_u[step][r].numpy())
    for a, b in zip(g_w, g_u):
        assert torch.equal(a.local.weights.data, b.local.weights.data)
        assert torch.equal(a.local.opt_state, b.local.opt_state)


def test_pull_transport_and_grad_requiring_weights_raise(host_peer_lib, monkeypatch):
    W, B = 2, 4
    cfgs, plan, spec, full, F, _, _, _, _ = _setup(W, True, 5)
    names = output_names_by_table(cfgs)
    ids = torch.zeros(F * B, dtype=torch.int64)
    off = torch.arange(F * B + 1, dtype=torch.int64)

    def run(mode, psw):
        monkeypatch.setenv("TZK_PEER_BWD", mode)
        registry, errs = {}, []

        def body(r, tbar):
            class St(M._sim_mixin(registry, tbar, mode), peer_exchange.PeerState):
                pass

            g = _DimGroup(cfgs, plan, r, W, torch.device("cpu"), True, names)
            g.local.set_optimizer(spec)
            st = St(g, plan, None, B)
            for fn in (lambda: st.gather(ids, off, psw), lambda: st.prep(ids, off, psw)):
                try:
                    fn()
                    errs.append("no error")
                except NotImplementedError as e:
                    errs.append(str(e))

        with Fn.use_backend(WeightedPeerSource(host_peer_lib)):
            M._run_ranks(W, body)
        return errs

    errs = run("pull", torch.ones(F * B))
    assert len(errs) == 2 * W and all("push" in e and "sharded" in e for e in errs), errs
    errs = run("push", torch.ones(F * B, requires_grad=True))
    assert len(errs) == 2 * W and all("require grad" in e for e in errs), errs
