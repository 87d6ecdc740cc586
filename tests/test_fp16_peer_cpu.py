"""FP16 tables (data_type = FP16) on sharded collections, without a GPU.

The peer-memory step (peer_exchange.PeerState + csrc/tzk_peer.cu) with every rank's arena and the local mirror of the
small tables held as halfs: W ranks run as threads of this process (tests/test_peer_exchange_model.py's plumbing), the
peer kernels as a loop-level model ("model") or from csrc/tzk_peer.cu compiled for the host ("source", with
tests/native/half_cpu_shim.h for the half type).  The owner's update is the oracle's fused update on the half arena:
fp32 arithmetic on the widened row, the new row rounded to the nearest half (ties to even).  Checked against the
unsharded FP16 collection stepped on the key-major concatenation of the W local batches (gradients / W):
  * the forward is bit-exact (SUM and MEAN, multi-hot bags with empty ones, weighted bags, sequences; one-launch and
    split gather; mirrored and remote tables);
  * dyadic data at W in {2, 4}: tables (halfs) and optimizer state bit-identical after three steps; otherwise tables
    within one fp16 ulp and the fp32 state within the fp32 peer tests' tolerance.
Also here: a dim group mixing FP32 and FP16 tables raises; the NCCL-exchange fallback (gloo) trains FP16 tables like
the unsharded model; checkpoints of FP16 tables move between W = 2, W = 1 and row-wise / table-wise plans, keep fp16
weights and fp32 state under the FP32 model's keys, and refuse to load across data_type."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import test_peer_exchange_model as M  # noqa: E402  (sets TZK_PEER_MIRROR_ROWS: some tables mirrored, some remote)
from oracle_backend import OracleKernels  # noqa: E402
from test_weighted_peer_cpu import WeightedPeerModel, WeightedPeerSource, _bags, _weights  # noqa: E402
from weighted_ref import WeightedOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200 import peer_exchange  # noqa: E402
from torcheasyrec_b200.distributed import TABLE_WISE, _DimGroup, make_plan  # noqa: E402
from torcheasyrec_b200.embedding_modules import (DataType, EmbeddingBagCollection, EmbeddingBagConfig,  # noqa: E402
                                                 EmbeddingCollection, EmbeddingConfig, SparseOptimizerSpec,
                                                 output_names_by_table)
from torcheasyrec_b200.kernels import OPT_ADAGRAD  # noqa: E402

P, I32, I64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
f32, f16 = np.float32, np.float16


@pytest.fixture(scope="module")
def host_peer_lib(tmp_path_factory):
    """csrc/tzk_peer.cu compiled for the host, with the FP16 entry points bound next to the fp32 ones."""
    exp = os.path.join(HERE, "native")
    out = str(tmp_path_factory.mktemp("f16shim") / "libtzk_peer_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", exp, "-x",
                    "c++", os.path.join(os.path.dirname(HERE), "torcheasyrec_b200", "csrc", "tzk_peer.cu"), "-shared",
                    "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    gather = [P, P, P, P, P, P, P, P, P, P, I32, I32, I32, I32, P, I64, P, P, P]
    L.tzk_peer_pooled_gather_fwd.argtypes = gather
    L.tzk_peer_pooled_gather_fwd_f16.argtypes = gather
    L.tzk_peer_pooled_gather_fwd_sel.argtypes = gather[:-1] + [P, I32, P]
    L.tzk_peer_pooled_gather_fwd_sel_f16.argtypes = gather[:-1] + [P, I32, P]
    L.tzk_peer_pooled_gather_fwd_weighted.argtypes = gather[:-1] + [P, P, I32, P]
    L.tzk_peer_pooled_gather_fwd_weighted_f16.argtypes = gather[:-1] + [P, P, I32, P]
    L.tzk_peer_seq_gather_fwd.argtypes = [P, P, P, P, P, P, P, I32, I32, I32, I32, I64, P, P, P, P]
    L.tzk_peer_seq_gather_fwd_f16.argtypes = [P, P, P, P, P, P, P, I32, I32, I32, I32, I64, P, P, P, P]
    L.tzk_peer_mirror_refresh.argtypes = [P, I32, P, P, P, P, I32, P, P]
    L.tzk_peer_mirror_refresh_f16.argtypes = [P, I32, P, P, P, P, I32, P, P]
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


def _is_f16(tables):
    return tables.t.dtype == torch.float16


def _p(t):
    return None if t is None else t.data_ptr()


class F16PeerSource(WeightedPeerSource):
    """The peer kernels from csrc/tzk_peer.cu's host-compiled source; half arenas go to the _f16 entry points."""

    name = "oracle+f16-peer-source"

    def peer_pooled_gather_fwd(self, tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets, B, W,
                               out=None, mirror=None, feat_mirror_off=None, feat_sel=None, per_sample_weights=None):
        if not _is_f16(tables):
            return super().peer_pooled_gather_fwd(tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets,
                                                  B, W, out, mirror, feat_mirror_off, feat_sel, per_sample_weights)
        assert mirror is None or mirror.dtype == torch.float16
        dim, col, pool = self._lay(lay)
        out = torch.full((B, lay.total_dim), float("nan")) if out is None else out
        args = [tables.ptrs, rf_w_off.data_ptr(), feat_rows.data_ptr(), feat_block.data_ptr(), feat_owner.data_ptr(),
                dim.data_ptr(), col.data_ptr(), pool.data_ptr(), ids.data_ptr(), offsets.data_ptr(), lay.num_features, B,
                W, (lay.max_dim + 3) // 4 * 4, out.data_ptr(), lay.total_dim, _p(mirror), _p(feat_mirror_off)]
        n_sel = 0 if feat_sel is None else feat_sel.numel()
        if per_sample_weights is not None and ids.numel():
            rc = self.L.tzk_peer_pooled_gather_fwd_weighted_f16(*args, per_sample_weights.data_ptr(), _p(feat_sel),
                                                                n_sel, None)
        elif feat_sel is not None:
            rc = self.L.tzk_peer_pooled_gather_fwd_sel_f16(*args, feat_sel.data_ptr(), n_sel, None)
        else:
            rc = self.L.tzk_peer_pooled_gather_fwd_f16(*args, None)
        assert rc == 0, rc
        return out

    def peer_seq_gather_fwd(self, tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets, B, W,
                            mirror=None, feat_mirror_off=None):
        if not _is_f16(tables):
            return super().peer_seq_gather_fwd(tables, rf_w_off, feat_rows, feat_block, feat_owner, lay, ids, offsets, B,
                                               W, mirror, feat_mirror_off)
        D, nnz = lay.dim[0], ids.numel()
        out = torch.full((nnz, D), float("nan"))
        rc = self.L.tzk_peer_seq_gather_fwd_f16(tables.ptrs, rf_w_off.data_ptr(), feat_rows.data_ptr(),
                                                feat_block.data_ptr(), feat_owner.data_ptr(), ids.data_ptr(),
                                                offsets.data_ptr(), lay.num_features, B, W, D, nnz, out.data_ptr(),
                                                _p(mirror), _p(feat_mirror_off), None)
        assert rc == 0, rc
        return out

    def peer_mirror_refresh(self, tables, W, seg_rank, seg_src, seg_dst, seg_n, mirror):
        if not _is_f16(tables):
            return super().peer_mirror_refresh(tables, W, seg_rank, seg_src, seg_dst, seg_n, mirror)
        assert mirror.dtype == torch.float16
        rc = self.L.tzk_peer_mirror_refresh_f16(tables.ptrs, W, seg_rank.data_ptr(), seg_src.data_ptr(),
                                                seg_dst.data_ptr(), seg_n.data_ptr(), seg_rank.numel(),
                                                mirror.data_ptr(), None)
        assert rc == 0, rc


def _backend(kernels, lib):
    return WeightedPeerModel() if kernels == "model" else F16PeerSource(lib)


def _fp16_configs():
    """M._pooled_configs() as FP16 tables: SUM and MEAN, one shared table, a 2-row table, a table-wise one."""
    return [EmbeddingBagConfig(num_embeddings=c.num_embeddings, embedding_dim=c.embedding_dim, name=c.name,
                               feature_names=list(c.feature_names), pooling=c.pooling, data_type=DataType.FP16)
            for c in M._pooled_configs()]


def _plan(cfgs, W, kind):
    if kind == "mixed":
        return make_plan(cfgs, W, "row_wise", {"t_tw": [TABLE_WISE], "t_tiny": [TABLE_WISE]})
    return make_plan(cfgs, W, kind)


def _setup(W, dyadic, seed, plan_kind="mixed", weighted=False, spec=None):
    rng = np.random.default_rng(seed)
    cfgs = _fp16_configs()
    B, D = 12, 16
    plan = _plan(cfgs, W, plan_kind)
    spec = spec or SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.05)
    with Fn.use_backend(OracleKernels()):
        full = EmbeddingBagCollection(cfgs, device="cpu")
        full.set_optimizer(spec)
    assert full.weights.dtype == torch.float16
    if dyadic:
        full.weights.data.copy_(torch.from_numpy((rng.integers(-16, 17, full.weights.numel()) / 16.0).astype(f16)))
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows, dyadic) for _ in range(W)]
    weights = [_weights(rng, b[0].numel(), dyadic) for b in batches] if weighted else None
    if dyadic:
        grads = [torch.from_numpy((rng.integers(-8, 9, (B, F * D)) / 8.0).astype(f32)) for _ in range(W)]
    else:
        grads = [torch.from_numpy(rng.standard_normal((B, F * D)).astype(f32)) for _ in range(W)]
    return cfgs, plan, spec, full, F, B, batches, weights, grads


def _shard(cfgs, plan, W, full, spec, pooled=True):
    names = output_names_by_table(cfgs)
    groups = []
    for r in range(W):
        g = _DimGroup(cfgs, plan, r, W, torch.device("cpu"), pooled, names)
        g.static_alpha = 2.5
        g.local.set_optimizer(spec)
        assert g.local.weights.dtype == torch.float16
        for t, c in enumerate(cfgs):
            n = g.local._table_rows[t]
            if n:
                start = 0 if plan[c.name].kind == TABLE_WISE else r * plan[c.name].block
                g.local.set_table_weight(t, full.table_weight(t)[start:start + n])
        groups.append(g)
    return groups


def _run_peer(cfgs, plan, W, B, spec, full, batches, weights, grads, backend, tag, steps):
    groups = _shard(cfgs, plan, W, full, spec)
    F = groups[0].F
    registry, outs = {}, [[None] * W for _ in range(steps)]
    states = [None] * W

    def body(r, tbar):
        class St(M._sim_mixin(registry, tbar, tag), peer_exchange.PeerState):
            pass

        st = states[r] = St(groups[r], plan, None, B, [B * 4] * F)
        ids, offs = batches[r]
        psw = None if weights is None else weights[r]
        for s in range(steps):
            outs[s][r] = st.gather(ids, offs, psw).clone()
            st.prep(ids, offs, psw)
            st.backward(grads[r], offs)

    with Fn.use_backend(backend):
        M._run_ranks(W, body)
    assert all(int(g.overflow.item()) == 0 for g in groups)
    for st in states:                        # halfs in the symmetric arena and the mirror; fp32 everywhere else
        assert st.tables.t.dtype == torch.float16
        assert st.mirror is None or st.mirror.dtype == torch.float16
        if st.small is not None:
            assert st.small["psum"].t.dtype == torch.float32
        if st.bwd_mode == "push":
            assert st.recv.t.dtype == torch.float32
    return groups, outs


def _gathered(groups, plan, cfgs, full, t, state=False):
    sh = plan[cfgs[t].name]
    src = full.table_state(t) if state else full.table_weight(t)
    got = torch.zeros_like(src)
    for r, g in enumerate(groups):
        n = g.local._table_rows[t]
        if n:
            start = 0 if sh.kind == TABLE_WISE else r * sh.block
            got[start:start + n] = g.local.table_state(t) if state else g.local.table_weight(t)
    return got


def assert_within_one_ulp(got, want, err_msg=""):
    """|got - want| <= one fp16 ulp of the larger magnitude (halfs compared as exact float64 values)."""
    g, w = got.numpy().astype(np.float64), want.numpy().astype(np.float64)
    ulp = np.spacing(np.maximum(np.abs(g), np.abs(w)).astype(f16)).astype(np.float64)
    bad = np.abs(g - w) > ulp
    assert not bad.any(), f"{err_msg}: {int(bad.sum())} elements more than one fp16 ulp apart, e.g. " \
                          f"{g[bad][:4]} vs {w[bad][:4]}"


def _check_against_unsharded(cfgs, plan, spec, full, F, B, W, batches, weights, grads, groups, outs, dyadic, steps):
    ref = WeightedOracleKernels()
    ids, offs = [b[0] for b in batches], [b[1] for b in batches]
    cat_ids, cat_off = M._cat_key_major(ids, offs, F, B, W)
    kw = {}
    if weights is not None:
        kw["per_sample_weights"] = torch.cat([weights[r][offs[r][f * B]:offs[r][(f + 1) * B]]
                                              for f in range(F) for r in range(W)])
    cat_grad = torch.cat(grads) / W
    for step in range(steps):
        for r in range(W):
            wkw = {} if weights is None else {"per_sample_weights": weights[r]}
            want = ref.pooled_gather_fwd(full.weights.data, full.layout, ids[r], offs[r], B, **wkw)
            if dyadic or step == 0:
                np.testing.assert_array_equal(outs[step][r].numpy(), want.numpy(), err_msg=f"step {step} rank {r}")
        ref.fused_bwd(spec.kind, True, cat_grad, full.weights.data, full.opt_state, full.layout, cat_ids, cat_off,
                      B * W, spec.lr, spec.eps, 1.0, **kw)
    for t, c in enumerate(cfgs):
        got = _gathered(groups, plan, cfgs, full, t)
        assert got.dtype == torch.float16
        st = _gathered(groups, plan, cfgs, full, t, state=True)
        assert st.dtype == torch.float32
        if dyadic:
            np.testing.assert_array_equal(got.numpy().view(np.uint16), full.table_weight(t).numpy().view(np.uint16),
                                          err_msg=c.name)
            np.testing.assert_array_equal(st.numpy(), full.table_state(t).numpy(), err_msg=c.name)
        else:
            assert_within_one_ulp(got, full.table_weight(t), c.name)
            np.testing.assert_allclose(st.numpy(), full.table_state(t).numpy(), rtol=5e-5, atol=1e-6, err_msg=c.name)


@pytest.mark.parametrize("kernels", ["model", "source"])
@pytest.mark.parametrize("small_bwd", ["1", "0"])
@pytest.mark.parametrize("W,dyadic", [(2, True), (4, True), (3, False), (4, False)])
def test_fp16_peer_step_matches_unsharded(W, dyadic, small_bwd, kernels, host_peer_lib, monkeypatch):
    """Three peer steps on half tables (mixed plan: row-wise + table-wise, mirrored + remote tables; SUM and MEAN,
    ragged bags with empty ones) against the unsharded FP16 step on the concatenated batch."""
    monkeypatch.setenv("TZK_PEER_SMALL_BWD", small_bwd)
    cfgs, plan, spec, full, F, B, batches, _, grads = _setup(W, dyadic, 60 + W + 10 * dyadic)
    groups, outs = _run_peer(cfgs, plan, W, B, spec, full, batches, None, grads, _backend(kernels, host_peer_lib),
                             "f16", 3)
    _check_against_unsharded(cfgs, plan, spec, full, F, B, W, batches, None, grads, groups, outs, dyadic, 3)


@pytest.mark.parametrize("kernels", ["model", "source"])
@pytest.mark.parametrize("W,dyadic", [(2, True), (3, False)])
def test_fp16_weighted_peer_step_matches_unsharded(W, dyadic, kernels, host_peer_lib):
    """Weighted bags on half tables: w * widened row pooled as the unsharded weighted f16 lookup; push of w * g."""
    cfgs, plan, spec, full, F, B, batches, weights, grads = _setup(W, dyadic, 90 + W, weighted=True)
    groups, outs = _run_peer(cfgs, plan, W, B, spec, full, batches, weights, grads, _backend(kernels, host_peer_lib),
                             "f16w", 3)
    _check_against_unsharded(cfgs, plan, spec, full, F, B, W, batches, weights, grads, groups, outs, dyadic, 3)


@pytest.mark.parametrize("kernels", ["model", "source"])
@pytest.mark.parametrize("plan_kind,W", [("row_wise", 3), ("table_wise", 3), ("row_wise", 4), ("table_wise", 2)])
def test_fp16_peer_plans(plan_kind, W, kernels, host_peer_lib):
    """Pure row-wise and pure table-wise plans (W in {2, 4}: dyadic data, bit-identical halfs; W = 3: random data,
    within one ulp — 1/3 is not dyadic)."""
    dyadic = W != 3
    cfgs, plan, spec, full, F, B, batches, _, grads = _setup(W, dyadic, 7 + W, plan_kind=plan_kind)
    groups, outs = _run_peer(cfgs, plan, W, B, spec, full, batches, None, grads, _backend(kernels, host_peer_lib),
                             "f16p", 2)
    _check_against_unsharded(cfgs, plan, spec, full, F, B, W, batches, None, grads, groups, outs, dyadic, 2)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("split", ["0", "1"])
def test_fp16_peer_forward_is_bit_identical(split, weighted, host_peer_lib, monkeypatch):
    """No update in between, the kernels' source: one-launch and split gather (mirrored features in one launch, remote
    ones in the other), plain and weighted bags — every output bit equals the unsharded FP16 lookup's."""
    monkeypatch.setenv("TZK_PEER_SPLIT_GATHER", split)
    W = 3
    cfgs, plan, spec, full, F, B, batches, weights, _ = _setup(W, False, 21, weighted=weighted)
    groups = _shard(cfgs, plan, W, full, spec)
    registry, outs, split_used = {}, [None] * W, [None] * W

    def body(r, tbar):
        class St(M._sim_mixin(registry, tbar, "fwd16"), peer_exchange.PeerState):
            pass

        st = St(groups[r], plan, None, B, [B * 4] * F)
        split_used[r] = st._split_lists() is not None
        outs[r] = st.gather(*batches[r], None if weights is None else weights[r])

    with Fn.use_backend(F16PeerSource(host_peer_lib)):
        M._run_ranks(W, body)
    assert all(s == (split == "1") for s in split_used)
    ref = WeightedOracleKernels()
    for r in range(W):
        wkw = {} if weights is None else {"per_sample_weights": weights[r]}
        want = ref.pooled_gather_fwd(full.weights.data, full.layout, batches[r][0], batches[r][1], B, **wkw)
        np.testing.assert_array_equal(outs[r].numpy(), want.numpy())


def test_fp16_mirror_refresh_copies_the_bits(host_peer_lib):
    """The FP16 mirror refresh at 8-B granularity: segments starting at odd multiples of 4 halfs (8-B but not 16-B
    aligned), NaN / inf / subnormal payloads, chunked and one-load-per-thread kernels."""
    rng = np.random.default_rng(3)
    W = 3
    arenas = [torch.from_numpy(rng.integers(0, 1 << 16, 20000, dtype=np.uint16).view(f16)) for _ in range(W)]
    segs = [(0, 4, 0, 12), (1, 12, 12, 8192 + 36), (2, 100, 8192 + 48, 4), (1, 4, 8192 + 52, 4096 * 3 + 4)]
    seg = [torch.tensor([s[i] for s in segs], dtype=torch.int32 if i == 0 else torch.int64) for i in range(4)]

    class T:
        t = arenas[0]
        ptrs = (ctypes.c_uint64 * W)(*[a.data_ptr() for a in arenas])

    for chunked in ("1", "0"):
        os.environ["TZK_PEER_MIRROR_CHUNKED"] = chunked
        try:
            mirror = torch.zeros(8192 + 52 + 4096 * 3 + 4 + 8, dtype=torch.float16)
            F16PeerSource(host_peer_lib).peer_mirror_refresh(T, W, *seg, mirror)
        finally:
            del os.environ["TZK_PEER_MIRROR_CHUNKED"]
        m = mirror.numpy().view(np.uint16)
        for r, s, d, n in segs:
            np.testing.assert_array_equal(m[d:d + n], arenas[r].numpy().view(np.uint16)[s:s + n])
        assert not m[8192 + 52 + 4096 * 3 + 4:].any()


@pytest.mark.parametrize("kernels", ["model", "source"])
@pytest.mark.parametrize("W", [2, 3])
def test_fp16_peer_sequence_collection(W, kernels, host_peer_lib):
    """EmbeddingCollection of half tables (un-pooled, ragged sequences): rows bit-equal to the unsharded FP16 lookup,
    tables after one update within one fp16 ulp of the unsharded FP16 step."""
    rng = np.random.default_rng(31 + W)
    mk = lambda n, rows, feats: EmbeddingConfig(num_embeddings=rows, embedding_dim=8, name=n, feature_names=feats,
                                                data_type=DataType.FP16)
    cfgs = [mk("q", 50, ["q_id"]), mk("s1", 211, ["seq_a"]), mk("s2", 40, ["seq_b"])]
    B, D, max_len = 7, 8, 6
    plan = make_plan(cfgs, W, "row_wise", {"s2": [TABLE_WISE]})
    spec = SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=0.1)
    with Fn.use_backend(OracleKernels()):
        full = EmbeddingCollection(cfgs, device="cpu")
        full.set_optimizer(spec)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = []
    for _ in range(W):
        lens = np.concatenate([np.ones(B, np.int64), rng.integers(0, max_len + 1, B), rng.integers(0, max_len + 1, B)])
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        ids = np.concatenate([rng.integers(0, feat_rows[b // B], lens[b]) for b in range(F * B)]).astype(np.int64)
        batches.append((torch.from_numpy(ids), torch.from_numpy(off)))
    grads = [torch.from_numpy(rng.standard_normal((b[0].numel(), D)).astype(f32)) for b in batches]
    groups = _shard(cfgs, plan, W, full, spec, pooled=False)
    registry, outs = {}, [None] * W

    def body(r, tbar):
        class St(M._sim_mixin(registry, tbar, "seq16"), peer_exchange.PeerState):
            pass

        st = St(groups[r], plan, None, B, [B, B * max_len, B * max_len])
        assert st.tables.t.dtype == torch.float16 and (st.mirror is None or st.mirror.dtype == torch.float16)
        outs[r] = st.gather(*batches[r])
        st.prep(*batches[r])
        st.backward(grads[r], batches[r][1])

    with Fn.use_backend(_backend(kernels, host_peer_lib)):
        M._run_ranks(W, body)
    k = OracleKernels()
    for r in range(W):
        np.testing.assert_array_equal(outs[r].numpy(), k.seq_gather_fwd(full.weights.data, full.layout, *batches[r],
                                                                        B).numpy())
    ids, offs = [b[0] for b in batches], [b[1] for b in batches]
    cat_ids, cat_off = M._cat_key_major(ids, offs, F, B, W)
    rows = [grads[r][offs[r][f * B]:offs[r][(f + 1) * B]] for f in range(F) for r in range(W)]
    k.fused_bwd(spec.kind, False, torch.cat(rows) / W, full.weights.data, full.opt_state, full.layout, cat_ids, cat_off,
                B * W, spec.lr, spec.eps, 1.0)
    for t, c in enumerate(cfgs):
        assert_within_one_ulp(_gathered(groups, plan, cfgs, full, t), full.table_weight(t), c.name)


def test_dim_group_mixing_fp32_and_fp16_raises():
    cfgs = [EmbeddingBagConfig(num_embeddings=30, embedding_dim=16, name="a", feature_names=["fa"],
                               data_type=DataType.FP16),
            EmbeddingBagConfig(num_embeddings=40, embedding_dim=16, name="b", feature_names=["fb"])]
    plan = make_plan(cfgs, 2, "row_wise")
    with Fn.use_backend(OracleKernels()):
        with pytest.raises(NotImplementedError, match="group them by data_type"):
            _DimGroup(cfgs, plan, 0, 2, torch.device("cpu"), True, output_names_by_table(cfgs))
        # one dtype per dim group is fine, also when the collection's dim groups differ in dtype
        g = _DimGroup(cfgs[:1], plan, 1, 2, torch.device("cpu"), True, output_names_by_table(cfgs[:1]))
        assert g.local.weights.dtype == torch.float16


# ---- whole models over gloo: the NCCL-exchange fallback and checkpoints ---------------------------------------------
def _nccl_fallback_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    try:
        from fp16_sharded_ref import verify_fp16_sharded

        with Fn.use_backend(OracleKernels()):
            verify_fp16_sharded("dlrm_criteo", "cpu", "mixed", exchange="nccl", rw_min_rows=200, bit_exact_logits=True)
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _spawn(world, target, *args):
    import torch.multiprocessing as mp
    from test_distributed_cpu import _free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, *args, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    bad = [(r, m) for r, m in res if m != "ok"]
    assert not bad, "\n".join(f"rank {r}: {m}" for r, m in bad)


@pytest.mark.parametrize("world", [2, 4])
def test_nccl_exchange_fallback_trains_fp16_tables(world):
    """exchange="nccl" (gloo here): the owners look rows up in and update their FP16 shards through the local
    collection — logits bit-equal to the unsharded FP16 model's, tables within one fp16 ulp after two steps."""
    _spawn(world, _nccl_fallback_worker)


def _ckpt_pipeline(sharding, seed, rw_min_rows, fp16=True):
    from fp16_sharded_ref import fp16_edits

    from torcheasyrec_b200.distributed import DenseGradSync, shard_model
    from torcheasyrec_b200.engine import Pipeline
    from torcheasyrec_b200.rank_models import dense_optimizer_from_config

    edits = fp16_edits("dlrm_criteo") if fp16 else None
    p = Pipeline("dlrm_criteo", device="cpu", max_rows=300, seed=seed, capturable=False, edits=edits)
    if sharding is not None:
        ref = Pipeline("dlrm_criteo", device="cpu", max_rows=300, seed=seed, capturable=False, edits=edits)
        shard_model(p.model, "cpu", default=sharding, rw_min_rows=rw_min_rows, source=ref.model)
        p.model.set_sparse_optimizer(ref.model.sparse_collections()[0].optimizer)
        p.dense_optimizer = dense_optimizer_from_config(p.cfg.train_config, p.model.dense_parameters())
        p.grad_sync = DenseGradSync(p.model.dense_parameters())
    return p


def _ckpt_worker(rank, world, port, tmp, phase, sharding, rw_min_rows, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    try:
        import torch.distributed.checkpoint as dcp
        from test_checkpoint_dcp import _dense_state, _full_tables

        from torcheasyrec_b200.checkpoint import list_checkpoint_keys, restore_model, save_model

        with Fn.use_backend(OracleKernels()):
            if phase == "save":
                p = _ckpt_pipeline(sharding, 5, rw_min_rows)
                for i in range(2):
                    p.eager_step(p.synthetic_batch(32, seed=10 + i + 100 * rank))
                save_model(tmp, p.model, p.dense_optimizer)
                w, s = _full_tables(p)
                assert all(v.dtype == torch.float16 for v in w.values()) and all(v.dtype == torch.float32
                                                                                for v in s.values())
                # the FP32 model writes the same keys
                p32 = _ckpt_pipeline(sharding, 5, rw_min_rows, fp16=False)
                p32.eager_step(p32.synthetic_batch(32, seed=10 + 100 * rank))     # (dense optimizer state)
                save_model(os.path.join(tmp, "fp32"), p32.model, p32.dense_optimizer)
                if rank == 0:
                    torch.save({"w": w, "s": s, "dense": {n: v.detach().clone() for n, v in p.model.named_parameters()
                                                          if not n.endswith(".weights")},
                                "adam": {k: v.clone() for k, v in _dense_state(p).items()}}, os.path.join(tmp, "expect.pt"))
                    keys = list_checkpoint_keys(tmp)
                    assert keys == list_checkpoint_keys(os.path.join(tmp, "fp32"))
                    meta = {}
                    for sub in ("model", "optimizer"):
                        meta.update(dcp.FileSystemReader(os.path.join(tmp, sub)).read_metadata().state_dict_metadata)
                    pre = "embedding_group.emb_impls.__BASE__.ebc.embedding_bags."
                    tables = [k for k in keys if k.startswith(pre) and k.endswith(".weight")]
                    assert tables and all(meta[k].properties.dtype == torch.float16 for k in tables)
                    moms = [k for k in keys if k.startswith("state." + pre) and k.endswith(".momentum1")]
                    assert moms and all(meta[k].properties.dtype == torch.float32 for k in moms)
            elif phase == "load":
                p = _ckpt_pipeline(sharding, 99, rw_min_rows)
                p.eager_step(p.synthetic_batch(32, seed=1 + rank))
                restore_model(tmp, p.model, p.dense_optimizer)
                exp = torch.load(os.path.join(tmp, "expect.pt"))
                w, s = _full_tables(p)
                for k in exp["w"]:
                    assert w[k].dtype == torch.float16
                    assert torch.equal(w[k].view(torch.int16), exp["w"][k].view(torch.int16)), k
                    assert torch.equal(s[k], exp["s"][k]), k
                for n, v in p.model.named_parameters():
                    if not n.endswith(".weights"):
                        assert torch.equal(v.detach(), exp["dense"][n]), n
                for k, v in _dense_state(p).items():
                    assert torch.equal(v, exp["adam"][k]), k
                p.eager_step(p.synthetic_batch(32, seed=3 + rank))
            else:                                 # across data_type: refused before anything is loaded
                p32 = _ckpt_pipeline(sharding, 99, rw_min_rows, fp16=False)
                before = _full_tables(p32)[0]
                with pytest.raises(ValueError, match="data_type"):
                    restore_model(tmp, p32.model, p32.dense_optimizer)
                after = _full_tables(p32)[0]
                assert all(torch.equal(before[k], after[k]) for k in before)
                p16 = _ckpt_pipeline(sharding, 99, rw_min_rows)
                with pytest.raises(ValueError, match="data_type"):
                    restore_model(os.path.join(tmp, "fp32"), p16.model, p16.dense_optimizer)
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("save_cfg,load_cfg", [((2, "mixed", 200), (1, None, 0)), ((1, None, 0), (2, "row_wise", 0)),
                                               ((2, "row_wise", 0), (2, "table_wise", 0))])
def test_fp16_checkpoint_round_trip_across_world_sizes_and_plans(tmp_path, save_cfg, load_cfg):
    """FP16 tables saved as fp16 row-sharded tensors under the FP32 model's keys, optimizer state as fp32; restored
    bit for bit under another world size / plan; a checkpoint of the other data_type is refused."""
    tmp = str(tmp_path)
    _spawn(save_cfg[0], _ckpt_worker, tmp, "save", save_cfg[1], save_cfg[2])
    _spawn(load_cfg[0], _ckpt_worker, tmp, "load", load_cfg[1], load_cfg[2])
    _spawn(load_cfg[0], _ckpt_worker, tmp, "cross", load_cfg[1], load_cfg[2])
