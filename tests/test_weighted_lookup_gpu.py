"""Weighted id features on the GPU: tzk_pooled_gather_fwd_weighted and the weighted fused backward against the weighted
reference (tests/weighted_ref.py), bit for bit where the data make every sum exact.

Exactness (as tests/test_fused_bwd_edges.py): gradients are k * 2^-6 with small nonzero k, weights come from
{+-0.25, +-0.5, 1, 2, 3}, grad_scale is a power of two and MEAN bags have 1, 2, 4 or 8 ids, so every contribution
grad_scale * w * g / L is a multiple of q = grad_scale * 2^-11 (2^-8 without MEAN bags).  While the absolute contributions of a row add up to less
than 2^24 q, every partial sum in any order is exact in fp32.  SGD with lr = -1 on a zero arena stores each row's sum,
so every touched row must equal its float64 sum bit for bit and every untouched row must stay 0.  Table values
k * 2^-4 make the weighted gather exact the same way.
"""
import copy
import os

import numpy as np
import pytest
import torch

from weighted_ref import WeightedOracleKernels, pooled_lookup_weighted

from torcheasyrec_b200 import functional as Fn
from torcheasyrec_b200.embedding_modules import (EmbeddingBagCollection, EmbeddingBagConfig, PoolingType,
                                                 SparseOptimizerSpec)
from torcheasyrec_b200.kernels import (OPT_ADAGRAD, OPT_ADAM, OPT_LAMB, OPT_LARS_SGD, OPT_PARTIAL_ROWWISE_ADAM,
                                       OPT_PARTIAL_ROWWISE_LAMB, OPT_ROWWISE_ADAGRAD, OPT_SGD, POOL_MEAN, POOL_SUM,
                                       FeatureLayout, build_layout, default_kernels)
from torcheasyrec_b200.sparse import KeyedJaggedTensor

pytestmark = pytest.mark.gpu
DEV = "cuda"
WSET = np.array([0.25, -0.25, 0.5, -0.5, 1.0, 2.0, 3.0], np.float32)
MEAN_LENS = (1, 2, 4, 8)
f32 = np.float32


def K():
    return default_kernels()


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---- gather ---------------------------------------------------------------------------------------------------------
def gather_case(rng, dims, pool, B, max_len, dyadic, rows=300):
    F = len(dims)
    if dyadic:
        tabs = [(rng.integers(-8, 9, size=(rows, d)) * 2.0 ** -4).astype(f32) for d in dims]
    else:
        tabs = [rng.standard_normal((rows, d)).astype(f32) for d in dims]
    L = rng.integers(0, max_len + 1, size=F * B).astype(np.int32)
    L[rng.random(F * B) < 0.15] = 0
    if pool == POOL_MEAN and dyadic:
        L = np.where(L > 0, rng.choice(MEAN_LENS, size=F * B), 0).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    ids = rng.integers(0, rows, size=int(off[-1])).astype(np.int64)
    ids[::11] = rows + 5                                        # out of range: reads row 0
    w = rng.choice(WSET, size=len(ids)) if dyadic else rng.standard_normal(len(ids)).astype(f32)
    return tabs, ids, off, w.astype(f32)


def arena_of(tabs, lay, dtype):
    a = torch.zeros(lay.arena_elems, dtype=torch.float32)
    for f, t in enumerate(tabs):
        st = lay.row_stride(f)
        v = a[lay.w_off[f]:lay.w_off[f] + t.shape[0] * st].view(t.shape[0], st)
        v[:, :t.shape[1]] = torch.from_numpy(t)
        if st > t.shape[1]:
            v[:, t.shape[1]:] = 7.0                              # the interleaved state half must never be read
    return a.to(dtype).to(DEV)


DIMS_BY_G = {1: [4], 2: [8], 4: [16, 12], 8: [32], 16: [64], 32: [128, 100]}


@pytest.mark.parametrize("fmt", ["dense", "interleaved", "fp16"])
@pytest.mark.parametrize("pool", [POOL_SUM, POOL_MEAN])
@pytest.mark.parametrize("g", sorted(DIMS_BY_G))
@pytest.mark.parametrize("misaligned", [False, True])
def test_gather_bit_exact_with_dyadic_data(fmt, pool, g, misaligned):
    rng = np.random.default_rng(g * 10 + pool)
    dims = DIMS_BY_G[g]
    B = 97
    tabs, ids, off, w = gather_case(rng, dims, pool, B, max_len=40, dyadic=True)
    lay = build_layout([t.shape[0] for t in tabs], dims, list(range(len(dims))), [pool] * len(dims),
                       interleaved=fmt == "interleaved").to(DEV)
    arena = arena_of(tabs, lay, torch.float16 if fmt == "fp16" else torch.float32)
    out = None
    if misaligned:         # a column slice one float in: VEC 1 on every G
        big = torch.zeros((B, lay.total_dim + 3), device=DEV)
        out = big[:, 1:1 + lay.total_dim]
    got = K().pooled_gather_fwd(arena, lay, cu(ids), cu(off), B, out=out, per_sample_weights=cu(w))
    ref = pooled_lookup_weighted(tabs, list(range(len(dims))), [pool] * len(dims), ids, off, B, w)
    assert got.cpu().numpy().tobytes() == np.ascontiguousarray(ref).tobytes()


def test_gather_long_and_empty_bags_and_random_data():
    rng = np.random.default_rng(9)
    dims = [16, 8, 36]
    B = 64
    for pool in (POOL_SUM, POOL_MEAN):
        tabs, ids, off, w = gather_case(rng, dims, pool, B, max_len=700, dyadic=False)
        lay = build_layout([t.shape[0] for t in tabs], dims, [0, 1, 2], [pool] * 3).to(DEV)
        got = K().pooled_gather_fwd(arena_of(tabs, lay, torch.float32), lay, cu(ids), cu(off), B,
                                    per_sample_weights=cu(w)).cpu().numpy()
        ref = pooled_lookup_weighted(tabs, [0, 1, 2], [pool] * 3, ids, off, B, w)
        np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-5 * np.abs(ref).max())
        L = np.diff(off)
        for f, c in enumerate(lay.col):
            assert np.all(got[L[f * B:(f + 1) * B] == 0, c:c + dims[f]] == 0)


@pytest.mark.parametrize("fmt", ["dense", "interleaved", "fp16"])
def test_gather_with_all_ones_weights_is_the_unweighted_gather(fmt):
    rng = np.random.default_rng(1)
    dims = [16, 4, 20]
    tabs, ids, off, _ = gather_case(rng, dims, POOL_MEAN, 300, max_len=9, dyadic=False)
    lay = build_layout([t.shape[0] for t in tabs], dims, [0, 1, 2], [POOL_MEAN, POOL_SUM, POOL_MEAN],
                       interleaved=fmt == "interleaved").to(DEV)
    arena = arena_of(tabs, lay, torch.float16 if fmt == "fp16" else torch.float32)
    a = K().pooled_gather_fwd(arena, lay, cu(ids), cu(off), 300, per_sample_weights=torch.ones(len(ids), device=DEV))
    b = K().pooled_gather_fwd(arena, lay, cu(ids), cu(off), 300)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- backward, exact row sums ------------------------------------------------------------------------------------------
TP = {1: 1024, 4: 256, 16: 64, 32: 32}           # tile size in sorted positions, 4096 / (4 G)
RUN_LENGTHS = (1, 2, 31, 32, 33, 255, 256, 257, 512, 513)


def run_case(rng, dim, pool, counts, kmax=3, wset=WSET, n_feat=2, rows=None):
    """Two features on one table; key i is hit counts[i] times (positions shuffled); every bag has 1 id (SUM) or 1, 2, 4
    or 8 ids (MEAN).  Returns (layout, ids, offsets, B, weights, grad, expected sums {row: float64 row})."""
    n = int(sum(counts))
    keys = np.repeat(np.arange(len(counts)), counts)
    rng.shuffle(keys)
    rows = rows or len(counts) + 3
    if pool == POOL_SUM:
        L = np.ones(n, np.int32)
    else:
        L = []
        left = n
        while left:
            x = int(rng.choice([m for m in MEAN_LENS if m <= left]))
            L.append(x)
            left -= x
        L = np.array(L, np.int32)
    nb = len(L)
    B = (nb + n_feat - 1) // n_feat
    L = np.concatenate([L, np.zeros(B * n_feat - nb, np.int32)])
    off = np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    lay = build_layout([rows], [dim], [0] * n_feat, [pool] * n_feat).to(DEV)
    grad = (rng.choice([k for k in range(-kmax, kmax + 1) if k], size=(B, lay.total_dim)) * 2.0 ** -6).astype(f32)
    w = rng.choice(wset, size=n).astype(f32)
    return lay, keys.astype(np.int64), off, B, w, grad


def expected(lay, ids, off, B, w, grad, gs):
    sums, mag = {}, {}
    for f in range(lay.num_features):
        c, D = lay.col[f], lay.dim[f]
        for b in range(B):
            s, e = int(off[f * B + b]), int(off[f * B + b + 1])
            for l in range(s, e):
                sc = gs * float(w[l]) / ((e - s) if lay.pool[f] == POOL_MEAN else 1)
                row = sc * grad[b, c:c + D].astype(np.float64)
                sums[int(ids[l])] = sums.get(int(ids[l]), 0.0) + row
                mag[int(ids[l])] = mag.get(int(ids[l]), 0.0) + np.abs(row)
    q = gs * 2.0 ** (-11 if POOL_MEAN in lay.pool else -8)     # SUM bags: no 1/L, the weights' 2^-2 only
    for r in mag:                                          # the exactness precondition of the module docstring
        assert np.all(mag[r] < 2 ** 24 * q)
        assert np.all(np.mod(sums[r] / q, 1.0) == 0)
    return sums


def readout(lay, ids, off, B, w, grad, gs=0.5, split=False, ws=None):
    arena = torch.zeros(lay.arena_elems, device=DEV)
    k = K()
    if split:
        ws = torch.empty(k.fused_bwd_workspace_bytes(lay, len(ids), weighted=True), dtype=torch.uint8, device=DEV)
        k.fused_bwd_sort(True, lay, cu(ids), cu(off), B, ws, per_sample_weights=cu(w))
        k.fused_bwd_apply(OPT_SGD, True, cu(grad), arena, None, lay, cu(off), len(ids), B, -1.0, 0.0, gs, ws,
                          per_sample_weights=cu(w))
    else:
        k.fused_bwd(OPT_SGD, True, cu(grad), arena, None, lay, cu(ids), cu(off), B, -1.0, 0.0, gs,
                    per_sample_weights=cu(w))
    torch.cuda.synchronize()
    return arena.cpu().numpy()


def assert_readout(lay, ids, off, B, w, grad, gs=0.5, **kw):
    sums = expected(lay, ids, off, B, w, grad, gs)
    got = readout(lay, ids, off, B, w, grad, gs, **kw)
    D = lay.dim[0]
    want = np.zeros_like(got)
    for r, s in sums.items():
        want[lay.w_off[0] + r * D:lay.w_off[0] + (r + 1) * D] = s.astype(f32)
    assert got.tobytes() == want.tobytes()


@pytest.fixture(params=["heads", "walk"])
def heads(request, monkeypatch):
    monkeypatch.setenv("TZK_BWD_HEADS", "1" if request.param == "heads" else "0")
    return request.param


@pytest.mark.parametrize("dim", [4, 16, 64, 128, 3, 260])
@pytest.mark.parametrize("pool", [POOL_SUM, POOL_MEAN])
def test_run_lengths_bit_exact(heads, dim, pool):
    rng = np.random.default_rng(dim + pool)
    g = min(32, max(1, 1 << (max(1, -(-dim // 4)) - 1).bit_length()))
    tp = TP.get(g, 4096 // (4 * g))
    counts = []
    for r in RUN_LENGTHS + (tp - 1, tp, tp + 1, 2 * tp + 1):
        counts += [1, r, int(rng.integers(1, 4))]
    lay, ids, off, B, w, grad = run_case(rng, dim, pool, counts)
    assert_readout(lay, ids, off, B, w, grad)


def test_tile_switch_falls_back_to_the_general_path(monkeypatch):
    monkeypatch.setenv("TZK_BWD_TILE", "1")
    rng = np.random.default_rng(3)
    lay, ids, off, B, w, grad = run_case(rng, 16, POOL_SUM, [1, 300, 2, 513, 1, 257])
    assert_readout(lay, ids, off, B, w, grad)


def test_hot_row_bit_exact():
    rng = np.random.default_rng(5)
    lay, ids, off, B, w, grad = run_case(rng, 16, POOL_SUM, [600_000, 3, 1, 2], kmax=1)
    assert_readout(lay, ids, off, B, w, grad)


def test_uint64_keys_bit_exact():
    """A table declared with 2^32 + 8 rows (64-bit sort keys); only its first rows exist in the arena and are hit."""
    rng = np.random.default_rng(6)
    counts = [1, 40, 2, 513, 3, 1]
    lay0, ids, off, B, w, grad = run_case(rng, 16, POOL_SUM, counts)
    rows = (1 << 32) + 8
    lay = FeatureLayout(w_off=lay0.w_off, rows=[rows, rows], dim=lay0.dim, col=lay0.col, pool=lay0.pool,
                        key_base=lay0.key_base, total_keys=rows, total_dim=lay0.total_dim,
                        arena_elems=lay0.arena_elems).to(DEV)
    assert_readout(lay, ids, off, B, w, grad)


@pytest.mark.parametrize("pool", [POOL_SUM, POOL_MEAN])
def test_split_sort_apply_equals_one_shot(pool):
    rng = np.random.default_rng(7 + pool)
    lay, ids, off, B, w, grad = run_case(rng, 16, pool, [1, 33, 2, 300, 1, 5, 257])
    assert_readout(lay, ids, off, B, w, grad, split=True)
    a = readout(lay, ids, off, B, w, grad, split=True)
    b = readout(lay, ids, off, B, w, grad)
    assert a.tobytes() == b.tobytes()


# ---- every optimizer, through the collection -----------------------------------------------------------------------
KINDS = {"sgd": OPT_SGD, "adagrad": OPT_ADAGRAD, "rowwise_adagrad": OPT_ROWWISE_ADAGRAD, "adam": OPT_ADAM,
         "partial_rowwise_adam": OPT_PARTIAL_ROWWISE_ADAM, "lamb": OPT_LAMB, "partial_rowwise_lamb": OPT_PARTIAL_ROWWISE_LAMB,
         "lars_sgd": OPT_LARS_SGD}


def collection(kind, device, pool, seed=0, fp16=False):
    torch.manual_seed(seed)
    from torcheasyrec_b200.embedding_modules import DataType

    cfgs = [EmbeddingBagConfig(num_embeddings=r, embedding_dim=d, name=f"t{i}", feature_names=[f"f{i}"],
                               pooling=PoolingType.MEAN if pool == POOL_MEAN else PoolingType.SUM,
                               data_type=DataType.FP16 if fp16 else DataType.FP32)
            for i, (r, d) in enumerate([(400, 16), (50, 8)])]
    ebc = EmbeddingBagCollection(cfgs, device=device)
    ebc.set_optimizer(SparseOptimizerSpec(kind=KINDS[kind], lr=0.05, eps=1e-3, beta1=0.8, beta2=0.9, weight_decay=0.01,
                                          initial_accumulator_value=0.1, momentum=0.5, eta=0.1, max_gradient=0.0))
    return ebc


def batch(rng, B=512, weights=True):
    L = rng.integers(0, 6, size=2 * B).astype(np.int32)
    ids = np.concatenate([rng.integers(0, (400, 50)[k // B], size=L[k]) for k in range(2 * B)]).astype(np.int64)
    w = rng.standard_normal(len(ids)).astype(f32) if weights else None
    grad = rng.standard_normal((B, 24)).astype(f32)
    return L, ids, w, grad


def step(ebc, L, ids, w, grad, device):
    kjt = KeyedJaggedTensor(["f0", "f1"], torch.from_numpy(ids).to(device), lengths=torch.from_numpy(L).to(device),
                            weights=None if w is None else torch.from_numpy(w).to(device))
    out = ebc(kjt).values()
    out.backward(torch.from_numpy(grad).to(device))
    if device == DEV:
        torch.cuda.synchronize()
    return out.detach().cpu()


def table_state(ebc):
    return [ebc.table_weight(t).detach().float().cpu().clone() for t in range(2)] + \
           [s.detach().cpu().clone() for t in range(2) for s in [ebc.table_state(t)] if s is not None]


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("pool", [POOL_SUM, POOL_MEAN])
def test_every_optimizer_weighted_against_the_reference(kind, pool):
    rng = np.random.default_rng(11)
    g, c = collection(kind, DEV, pool), collection(kind, "cpu", pool)
    c.load_state_dict({k: v.cpu() for k, v in g.state_dict().items()})
    for it in range(2):
        L, ids, w, grad = batch(rng)
        og = step(g, L, ids, w, grad, DEV)
        with Fn.use_backend(WeightedOracleKernels()):
            oc = step(c, L, ids, w, grad, "cpu")
        np.testing.assert_allclose(og.numpy(), oc.numpy(), rtol=1e-5, atol=1e-6)
    for a, b in zip(table_state(g), table_state(c)):
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_all_ones_weights_update_is_the_unweighted_update(kind):
    """Default layout: element-wise Adagrad uses the interleaved [weight | accumulator] arena."""
    res = []
    for weighted in (True, False):
        rng = np.random.default_rng(12)
        ebc = collection(kind, DEV, POOL_MEAN, seed=4)
        for it in range(2):
            L, ids, _, grad = batch(rng, weights=False)
            step(ebc, L, ids, np.ones(len(ids), f32) if weighted else None, grad, DEV)
        res.append(table_state(ebc))
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(res[0], res[1]))


def test_fp16_tables_weighted():
    rng = np.random.default_rng(13)
    g, c = collection("adagrad", DEV, POOL_SUM, fp16=True), collection("adagrad", "cpu", POOL_SUM, fp16=True)
    c.load_state_dict({k: v.cpu() for k, v in g.state_dict().items()})
    L, ids, w, grad = batch(rng)
    og = step(g, L, ids, w, grad, DEV)
    with Fn.use_backend(WeightedOracleKernels()):
        c.weights.data = c.weights.data.float()          # the numpy oracle works on fp32 rows; round back below
        oc = step(c, L, ids, w, grad, "cpu")
    np.testing.assert_allclose(og.numpy(), oc.numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(g.weights.detach().float().cpu().numpy(), c.weights.data.half().float().numpy(),
                               rtol=1e-3, atol=1e-3)


# ---- the CUDA graph on the Ali-CCP MMoE config --------------------------------------------------------------------------
CCP_MMOE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_examples", "mmoe_taobao_ccp.config")
NO_DROPOUT = {"model_config.mmoe.task_towers[0].mlp.dropout_ratio": [],
              "model_config.mmoe.task_towers[1].mlp.dropout_ratio": [], "model_config.mmoe.expert_mlp.dropout_ratio": []}


def test_graphed_ccp_mmoe_replay_equals_eager_and_matches_the_reference():
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    a = Pipeline(CCP_MMOE, device="cuda:0", max_rows=1000, seed=3, edits=NO_DROPOUT)
    batches = [a.synthetic_batch(1024, seed=40 + i) for i in range(3)]
    assert all(next(iter(b.sparse_features.values())).weights_or_none() is not None for b in batches)
    step_g = GraphedTrainStep(a, batches[0], warmup=2)
    b = Pipeline(CCP_MMOE, device="cuda:0", max_rows=1000, seed=3, edits=NO_DROPOUT)
    b.model.load_state_dict(a.model.state_dict())
    for ca, cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
        if ca.layout.interleaved:
            cb.weights.data.copy_(ca.weights.data)
        else:
            cb.opt_state.copy_(ca.opt_state)
    b.dense_optimizer.load_state_dict(copy.deepcopy(a.dense_optimizer.state_dict()))
    for bt in batches[1:]:                 # new ids AND new weights each replay
        step_g.load(bt.pin_memory())
        la = float(step_g.replay())
        lb = float(b.eager_step(bt.to("cuda:0")))
        assert la == lb
    for ca, cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
        assert torch.equal(ca.weights.data.view(torch.int32), cb.weights.data.view(torch.int32))

    # one step against the oracle-backed CPU step (DESIGN §5 tolerances)
    gpu = Pipeline(CCP_MMOE, device="cuda:0", max_rows=1000, seed=11, edits=NO_DROPOUT, capturable=False)
    cpu = Pipeline(CCP_MMOE, device="cpu", max_rows=1000, seed=11, edits=NO_DROPOUT)
    cpu.model.load_state_dict({k: v.cpu() for k, v in gpu.model.state_dict().items()})
    bt = gpu.synthetic_batch(256, seed=5)
    lg = float(gpu.eager_step(bt.to("cuda:0")))
    with Fn.use_backend(WeightedOracleKernels()):
        lc = float(cpu.eager_step(bt))
    assert abs(lg - lc) <= 1e-5 * max(1.0, abs(lc))
    for cg, cc in zip(gpu.model.sparse_collections(), cpu.model.sparse_collections()):
        np.testing.assert_allclose(cg.dense_weights().cpu().numpy(), cc.dense_weights().numpy(), rtol=1e-4, atol=1e-6)
