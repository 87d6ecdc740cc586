"""Weighted id features without a GPU: the weighted reference, the host plumbing (KJT permute, DataParser, the lookup's
autograd function, sharded collections) and CPU training of the Ali-CCP MMoE config through the test backend."""
import os

import numpy as np
import pytest
import torch

from oracle import tzk_oracle as O
from sparse_optim_ref import OPT_LAMB, OPT_LARS_SGD, OPT_PARTIAL_ROWWISE_LAMB, WD_L2
from weighted_ref import WeightedOracleKernels, pooled_lookup_weighted

from torcheasyrec_b200 import functional as Fn
from torcheasyrec_b200.embedding_modules import (EmbeddingBagCollection, EmbeddingBagConfig, PoolingType,
                                                 SparseOptimizerSpec)
from torcheasyrec_b200.kernels import (OPT_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM, OPT_ROWWISE_ADAGRAD, OPT_SGD,
                                       build_layout)
from torcheasyrec_b200.sparse import KeyedJaggedTensor

CCP_MMOE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_examples", "mmoe_taobao_ccp.config")
CCP_WEIGHTED = ["user_shop", "user_brand", "user_intent", "user_cate", "item_user_intentid", "cross_user_shop_item_shopid",
                "cross_user_brand_item_brandid", "cross_user_intent_item_user_intentid", "cross_user_cate_item_cateid"]
f32 = np.float32


def bags(rng, F, B, max_len=5, p_empty=0.2):
    L = rng.integers(1, max_len + 1, size=F * B)
    L[rng.random(F * B) < p_empty] = 0
    return L.astype(np.int32)


def case(seed, dims=(4, 8), rows=(7, 5), B=6):
    rng = np.random.default_rng(seed)
    tables = [rng.standard_normal((r, d)).astype(f32) for r, d in zip(rows, dims)]
    ft = list(range(len(dims)))
    L = bags(rng, len(ft), B)
    off = O.lengths_to_offsets(L)
    ids = np.concatenate([rng.integers(0, rows[ft[k // B]], size=L[k]) for k in range(len(L))]).astype(np.int64)
    ids[::3] = 1                                                   # repeated ids inside and across bags
    w = rng.standard_normal(len(ids)).astype(f32)                 # negative weights too
    return tables, ft, ids, off, w, B


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_weighted_sum_matches_torch_embedding_bag(seed):
    tables, ft, ids, off, w, B = case(seed)
    out = pooled_lookup_weighted(tables, ft, [O.POOL_SUM] * len(ft), ids, off, B, w)
    col = 0
    for f, t in enumerate(ft):
        s, e = off[f * B], off[(f + 1) * B]
        ref = torch.nn.functional.embedding_bag(torch.from_numpy(ids[s:e]), torch.from_numpy(tables[t]),
                                                torch.from_numpy(off[f * B:(f + 1) * B] - s),
                                                per_sample_weights=torch.from_numpy(w[s:e]), mode="sum")
        D = tables[t].shape[1]
        np.testing.assert_allclose(out[:, col:col + D], ref.numpy(), rtol=1e-6, atol=1e-6)
        assert np.all(out[np.diff(off[f * B:(f + 1) * B + 1]) == 0, col:col + D] == 0)   # empty bags give 0
        col += D


def test_weighted_mean_against_float64():
    tables, ft, ids, off, w, B = case(5)
    out = pooled_lookup_weighted(tables, ft, [O.POOL_MEAN] * len(ft), ids, off, B, w)
    col = 0
    for f, t in enumerate(ft):
        D = tables[t].shape[1]
        for b in range(B):
            s, e = off[f * B + b], off[f * B + b + 1]
            ref = np.zeros(D)
            for l in range(s, e):
                ref += float(w[l]) * tables[t][ids[l]].astype(np.float64)
            if e > s:
                ref /= e - s
            np.testing.assert_allclose(out[b, col:col + D], ref, rtol=2e-6, atol=2e-6)
        col += D


@pytest.mark.parametrize("pool", [O.POOL_SUM, O.POOL_MEAN])
def test_all_ones_weights_equal_the_unweighted_oracle_bit_for_bit(pool):
    tables, ft, ids, off, _, B = case(7)
    ones = np.ones(len(ids), f32)
    a = pooled_lookup_weighted(tables, ft, [pool] * len(ft), ids, off, B, ones)
    b = O.pooled_lookup(tables, ft, [pool] * len(ft), ids, off, B)
    assert a.tobytes() == b.tobytes()


# ---- the weighted fused update: the backend against an independent float64 statement ---------------------------------
KINDS = {"sgd": OPT_SGD, "adagrad": OPT_ADAGRAD, "rowwise_adagrad": OPT_ROWWISE_ADAGRAD, "adam": OPT_ADAM,
         "partial_rowwise_adam": OPT_PARTIAL_ROWWISE_ADAM, "lamb": OPT_LAMB, "partial_rowwise_lamb": OPT_PARTIAL_ROWWISE_LAMB,
         "lars_sgd": OPT_LARS_SGD, "rowwise_adagrad_l2": OPT_ROWWISE_ADAGRAD}


def collection(dims, rows, pool, kind_name, seed=0):
    torch.manual_seed(seed)
    cfgs = [EmbeddingBagConfig(num_embeddings=r, embedding_dim=d, name=f"t{i}", feature_names=[f"f{i}"],
                               pooling=PoolingType.MEAN if pool == O.POOL_MEAN else PoolingType.SUM)
            for i, (r, d) in enumerate(zip(rows, dims))]
    ebc = EmbeddingBagCollection(cfgs, device="cpu")
    kw = dict(lr=0.05, eps=1e-3, beta1=0.8, beta2=0.9, weight_decay=0.01)
    if kind_name == "rowwise_adagrad_l2":
        kw["weight_decay_mode"] = WD_L2
    if kind_name == "lars_sgd":
        kw.update(momentum=0.5, eta=0.1)
    ebc.set_optimizer(SparseOptimizerSpec(kind=KINDS[kind_name], initial_accumulator_value=0.1, **kw))
    return ebc


def f64_update(kind_name, w, g, m, v, spec, step):
    """Float64 statement of one update of rows w from their summed gradients g."""
    lr, eps, b1, b2, wd = spec.lr, spec.eps, spec.beta1, spec.beta2, spec.weight_decay
    D = w.shape[1]
    sq = lambda x: (x * x).sum(axis=1)
    if kind_name == "sgd":
        return w - lr * g, m, v
    if kind_name == "adagrad":
        m = m + g * g
        return w - lr * g / (np.sqrt(m) + eps), m, v
    if kind_name in ("rowwise_adagrad", "rowwise_adagrad_l2"):
        if kind_name == "rowwise_adagrad":
            v = v + sq(g) / D
            return w - lr * g / (np.sqrt(v) + eps)[:, None], m, v
        v = v + sq(g + wd * w) / D
        mult = lr / (np.sqrt(v) + eps)
        return (1 - mult * wd)[:, None] * w - mult[:, None] * g, m, v
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    if kind_name in ("adam", "partial_rowwise_adam", "lamb", "partial_rowwise_lamb"):
        m = b1 * m + (1 - b1) * g
        if kind_name in ("adam", "lamb"):
            v = b2 * v + (1 - b2) * g * g
            den = np.sqrt(v / bc2) + eps
        else:
            v = b2 * v + (1 - b2) * sq(g) / D
            den = (np.sqrt(v / bc2) + eps)[:, None]
        if kind_name.endswith("adam"):
            return w - lr * ((m / bc1) / den + wd * w), m, v
        u = (m / bc1) / den + wd * w
        return w - (lr * np.sqrt(sq(w)) / np.sqrt(sq(u)))[:, None] * u, m, v
    # lars_sgd
    wn = np.sqrt(sq(w))
    lr_r = lr * spec.eta * wn / (np.sqrt(sq(g)) + wd * wn)
    m = spec.momentum * m + lr_r[:, None] * (g + wd * w)
    return w - m, m, v


@pytest.mark.parametrize("kind_name", sorted(KINDS))
@pytest.mark.parametrize("pool", [O.POOL_SUM, O.POOL_MEAN])
def test_weighted_update_of_every_kind_against_float64(kind_name, pool):
    rng = np.random.default_rng(3)
    dims, rows, B = (4, 8), (6, 5), 7
    ebc = collection(dims, rows, pool, kind_name)
    L = bags(rng, 2, B, max_len=4)
    off = O.lengths_to_offsets(L)
    ids = np.concatenate([rng.integers(0, rows[k // B], size=L[k]) for k in range(len(L))]).astype(np.int64)
    psw = rng.standard_normal(len(ids)).astype(f32)
    w0 = [ebc.table_weight(t).clone().numpy().astype(np.float64) for t in range(2)]
    kjt = KeyedJaggedTensor(["f0", "f1"], torch.from_numpy(ids), lengths=torch.from_numpy(L), weights=torch.from_numpy(psw))
    grad = rng.standard_normal((B, sum(dims))).astype(f32)
    with Fn.use_backend(WeightedOracleKernels()):
        out = ebc(kjt).values()
        out.backward(torch.from_numpy(grad))
    spec = ebc.optimizer
    col = 0
    for t in range(2):
        D = dims[t]
        gsum = {}
        for b in range(B):
            s, e = off[t * B + b], off[t * B + b + 1]
            for l in range(s, e):
                sc = float(psw[l]) / ((e - s) if pool == O.POOL_MEAN else 1)
                gsum[ids[l]] = gsum.get(ids[l], 0.0) + sc * grad[b, col:col + D].astype(np.float64)
        uniq = np.array(sorted(gsum))
        g = np.stack([gsum[i] for i in uniq])
        st = ebc.table_state(t)
        m = np.zeros_like(g) if kind_name not in ("adagrad",) else np.full_like(g, 0.1)
        v = np.full(len(uniq), 0.1) if "rowwise_adagrad" in kind_name else (
            np.zeros_like(g) if kind_name in ("adam", "lamb") else np.zeros(len(uniq)))
        ref, _, _ = f64_update(kind_name, w0[t][uniq], g, m, v, spec, 1)
        got = ebc.table_weight(t).numpy()[uniq]
        np.testing.assert_allclose(got, ref, rtol=2e-4, atol=2e-6)
        untouched = np.setdiff1d(np.arange(rows[t]), uniq)
        np.testing.assert_array_equal(ebc.table_weight(t).numpy()[untouched], w0[t][untouched].astype(f32))
        assert st is None or st.shape[0] == rows[t]
        col += D


def test_all_ones_weighted_update_equals_the_unweighted_update_bit_for_bit():
    rng = np.random.default_rng(4)
    B = 9
    L = bags(rng, 2, B)
    off = O.lengths_to_offsets(L)
    ids = np.concatenate([rng.integers(0, (6, 5)[k // B], size=L[k]) for k in range(len(L))]).astype(np.int64)
    grad = torch.from_numpy(rng.standard_normal((B, 12)).astype(f32))
    res = []
    for weights in (torch.ones(len(ids)), None):
        ebc = collection((4, 8), (6, 5), O.POOL_MEAN, "adam", seed=2)
        kjt = KeyedJaggedTensor(["f0", "f1"], torch.from_numpy(ids), lengths=torch.from_numpy(L), weights=weights)
        with Fn.use_backend(WeightedOracleKernels()):
            ebc(kjt).values().backward(grad)
        res.append(np.concatenate([ebc.table_weight(t).numpy().ravel() for t in range(2)] +
                                  [ebc.table_state(t).numpy().ravel() for t in range(2)]))
    assert res[0].tobytes() == res[1].tobytes()          # (the arena's padding tail is never initialised)


# ---- host plumbing ----------------------------------------------------------------------------------------------------
def test_kjt_permute_carries_the_weights():
    rng = np.random.default_rng(0)
    B = 4
    L = bags(rng, 3, B)
    ids = torch.arange(int(L.sum()), dtype=torch.int64)
    w = torch.from_numpy(rng.standard_normal(int(L.sum())).astype(f32))
    kjt = KeyedJaggedTensor(["a", "b", "c"], ids, lengths=torch.from_numpy(L), weights=w)
    with Fn.use_backend(WeightedOracleKernels()):
        p = kjt.permute([2, 0, 2])
    assert p.keys() == ["c", "a", "c"]
    # ids are positions here, so the permuted ids index the weight each position must carry
    assert torch.equal(p.weights_or_none(), w[p.values()])
    with Fn.use_backend(WeightedOracleKernels()):
        assert kjt.permute([0, 1]).weights_or_none() is not None
        assert KeyedJaggedTensor(["a"], ids[:2], lengths=torch.tensor([2, 0, 0, 0], dtype=torch.int32)
                                 ).permute([0]).weights_or_none() is None


def test_weights_that_require_grad_raise():
    ebc = collection((4,), (5,), O.POOL_SUM, "sgd")
    kjt = KeyedJaggedTensor(["f0"], torch.tensor([1, 2]), lengths=torch.tensor([2], dtype=torch.int32),
                            weights=torch.ones(2, requires_grad=True))
    with Fn.use_backend(WeightedOracleKernels()), pytest.raises(NotImplementedError, match="require grad"):
        ebc(kjt)


def test_c_oracle_raises_on_weighted_input():
    from oracle import c_oracle

    if not c_oracle.available():
        pytest.skip("the C oracle is not built")
    k = WeightedOracleKernels(use_c=True)
    lay = build_layout([5], [4], [0], [0])
    w = torch.zeros(lay.arena_elems)
    with pytest.raises(NotImplementedError, match="C oracle"):
        k.pooled_gather_fwd(w, lay, torch.tensor([1]), torch.tensor([0, 1]), 1, per_sample_weights=torch.ones(1))


def _gloo_sharded_raises(rank, world, port, q):
    import torch.distributed as dist

    from torcheasyrec_b200.distributed import ShardedEmbeddingBagCollection, TableShard

    try:
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
        cfg = EmbeddingBagConfig(num_embeddings=8, embedding_dim=4, name="t0", feature_names=["f0"])
        plan = {"t0": TableShard(kind="row_wise", block=4)}
        sm = ShardedEmbeddingBagCollection([cfg], plan, torch.device("cpu"))
        kjt = KeyedJaggedTensor(["f0"], torch.tensor([1, 6]), lengths=torch.tensor([1, 1], dtype=torch.int32),
                                weights=torch.ones(2))
        try:
            sm(kjt)
            q.put((rank, "no error"))
        except NotImplementedError as e:
            q.put((rank, "raised" if "sharded" in str(e) else str(e)))
    except Exception as e:      # reported to the parent, which fails the test
        q.put((rank, repr(e)))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def test_sharded_collection_raises_on_weighted_kjt():
    import socket

    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_gloo_sharded_raises, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = dict(q.get(timeout=120) for _ in ps)
    for p in ps:
        p.join(timeout=60)
    assert res == {0: "raised", 1: "raised"}, res


def test_data_parser_to_embedding_group_with_weighted_and_unweighted_keys():
    from torcheasyrec_b200.engine import Pipeline

    edits = {"model_config.mmoe.task_towers[0].mlp.dropout_ratio": [], "model_config.mmoe.task_towers[1].mlp.dropout_ratio": [],
             "model_config.mmoe.expert_mlp.dropout_ratio": []}
    p = Pipeline(CCP_MMOE, device="cpu", max_rows=50, seed=2, edits=edits)
    weighted = sorted(f.name for f in p.features if f.is_weighted)
    assert weighted == sorted(CCP_WEIGHTED)
    from torcheasyrec_b200.data_parser import DataParser

    parser = DataParser(p.features, p.labels)
    B = 3
    rng = np.random.default_rng(1)
    data = {}
    for f in p.features:
        if f.is_sparse:
            L = torch.from_numpy(rng.integers(0, 3, size=B).astype(np.int32))
            data[f"{f.name}.values"] = torch.from_numpy(rng.integers(0, 50, size=int(L.sum())).astype(np.int64))
            data[f"{f.name}.lengths"] = L
            if f.is_weighted:
                data[f"{f.name}.weights"] = torch.from_numpy(rng.random(int(L.sum())).astype(f32))
        else:
            data[f"{f.name}.values"] = torch.from_numpy(rng.random((B, f.value_dim)).astype(f32))
    for name in p.labels:
        data[name] = torch.zeros(B)
    batch = parser.to_batch(data)
    (kjt,) = batch.sparse_features.values()
    w = kjt.weights_or_none()
    assert w is not None and w.numel() == kjt.values().numel()
    o = 0
    for key, n in zip(kjt.keys(), kjt.length_per_key()):
        if key in CCP_WEIGHTED:
            assert torch.equal(w[o:o + n], data[f"{key}.weights"])
        else:
            assert torch.all(w[o:o + n] == 1)
        o += n
    with Fn.use_backend(WeightedOracleKernels()):
        emb = p.model.embedding_group(batch)
        # the weighted bags are pooled with their weights: scaling every weight by 2 doubles those columns only
        batch2 = parser.to_batch({k: (v * 2 if k.endswith(".weights") else v) for k, v in data.items()})
        emb2 = p.model.embedding_group(batch2)
    (g,) = emb.keys()
    assert not torch.equal(emb[g], emb2[g])
    assert torch.allclose(emb2[g][emb2[g] != emb[g]], 2 * emb[g][emb2[g] != emb[g]], rtol=1e-5, atol=1e-6)


def test_ccp_mmoe_trains_on_cpu_through_the_test_backend():
    from torcheasyrec_b200.engine import Pipeline

    edits = {"model_config.mmoe.task_towers[0].mlp.dropout_ratio": [], "model_config.mmoe.task_towers[1].mlp.dropout_ratio": [],
             "model_config.mmoe.expert_mlp.dropout_ratio": []}
    p = Pipeline(CCP_MMOE, device="cpu", max_rows=200, seed=3, edits=edits)
    losses = []
    with Fn.use_backend(WeightedOracleKernels()):
        for s in range(3):
            b = p.synthetic_batch(64, seed=s)
            assert next(iter(b.sparse_features.values())).weights_or_none() is not None
            losses.append(float(p.eager_step(b)))
    assert all(np.isfinite(losses))
