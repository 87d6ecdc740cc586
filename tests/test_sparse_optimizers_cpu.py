"""LAMB, partial row-wise LAMB, LARS-SGD and row-wise Adagrad's weight-decay modes on the host: the numpy reference
(tests/sparse_optim_ref.py) against an independent float64 statement and against invariants of the formulas, the
train_config mapping, checkpoint keys and DCP round trips, and CPU training steps with the reference as compute."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import tzk_oracle as O  # noqa: E402
from sparse_optim_ref import (OPT_LAMB, OPT_LARS_SGD, OPT_PARTIAL_ROWWISE_LAMB, WD_DECOUPLE, WD_L2,  # noqa: E402
                              ExtOracleKernels, update_rows)
from test_distributed_cpu import _free_port  # noqa: E402

from torcheasyrec_b200 import kernels as K  # noqa: E402

U = 2.0 ** -24
KINDS = {"lamb": OPT_LAMB, "partial_rowwise_lamb": OPT_PARTIAL_ROWWISE_LAMB, "lars_sgd": OPT_LARS_SGD}


def test_constants_match_the_package():
    assert (K.OPT_LAMB, K.OPT_PARTIAL_ROWWISE_LAMB, K.OPT_LARS_SGD) == (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB, OPT_LARS_SGD)
    assert (K.WD_NONE, K.WD_L2, K.WD_DECOUPLE) == (0, WD_L2, WD_DECOUPLE) and K.LARS_ETA == 0.001
    assert K.norm_family(K.OPT_LAMB, {}) and K.norm_family(K.OPT_LARS_SGD, {})
    assert K.norm_family(K.OPT_ROWWISE_ADAGRAD, dict(weight_decay=0.1, weight_decay_mode=WD_L2))
    assert not K.norm_family(K.OPT_ROWWISE_ADAGRAD, dict(weight_decay=0.0, weight_decay_mode=WD_L2))
    assert not K.norm_family(K.OPT_ROWWISE_ADAGRAD, dict(weight_decay=0.1, weight_decay_mode=0))
    assert not K.norm_family(K.OPT_ADAM, dict(weight_decay=0.1))


# ---- float64 statement of the formulas (independent of the reference's operation order) ----------------------------
def f64_update(opt, w, g, m, v, p, mode=0):
    lr, eps, wd = p["lr"], p["eps"], p["weight_decay"]
    D = w.shape[1]
    if opt in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB):
        b1, b2, t = p["beta1"], p["beta2"], p["step"]
        m = b1 * m + (1 - b1) * g
        if opt == OPT_LAMB:
            v = b2 * v + (1 - b2) * g * g
            vh = v / (1 - b2 ** t)
        else:
            v = b2 * v + (1 - b2) * np.mean(g * g, axis=1)
            vh = (v / (1 - b2 ** t))[:, None]
        u = (m / (1 - b1 ** t)) / (np.sqrt(vh) + eps) + wd * w
        ratio = np.linalg.norm(w, axis=1) / np.linalg.norm(u, axis=1)
        return w - lr * ratio[:, None] * u, m, v
    if opt == OPT_LARS_SGD:
        wn, gn = np.linalg.norm(w, axis=1), np.linalg.norm(g, axis=1)
        lr_r = lr * p["eta"] * wn / (gn + wd * wn)
        m = p["momentum"] * m + lr_r[:, None] * (g + wd * w)
        return w - m, m, v
    gl = g + wd * w if mode == WD_L2 else g
    s = v + np.sum(gl * gl, axis=1) / D
    mult = (lr / (np.sqrt(s) + eps))[:, None]
    keep = 1 - mult * wd if mode == WD_L2 else 1 - lr * wd
    return keep * w - mult * g, m, s


P = dict(lr=0.05, eps=1e-8, beta1=0.8, beta2=0.95, weight_decay=0.01, step=3, momentum=0.7, eta=0.01)


@pytest.mark.parametrize("name,mode", [("lamb", 0), ("partial_rowwise_lamb", 0), ("lars_sgd", 0),
                                       ("rowwise_adagrad_l2", WD_L2), ("rowwise_adagrad_decouple", WD_DECOUPLE)])
@pytest.mark.parametrize("D", [1, 4, 16, 129])
def test_reference_matches_float64_statement(name, mode, D):
    """Random rows: every output within a few hundred fp32 ulps (relative) of the float64 statement; the norms add up D
    squares (relative error <= D u each), which the bound grows with."""
    rng = np.random.default_rng(D * 10 + mode)
    n = 37
    w = rng.standard_normal((n, D)).astype(np.float32)
    g = (rng.standard_normal((n, D)) * 0.1).astype(np.float32)
    opt = KINDS.get(name, O.OPT_ROWWISE_ADAGRAD)
    m = (rng.standard_normal((n, D)) * 0.01).astype(np.float32) if opt != O.OPT_ROWWISE_ADAGRAD else None
    if opt == OPT_LAMB:
        v = (rng.random((n, D)) * 0.01).astype(np.float32)
    elif opt in (OPT_PARTIAL_ROWWISE_LAMB, O.OPT_ROWWISE_ADAGRAD):
        v = (rng.random(n) * 0.01).astype(np.float32)
    else:
        v = None
    got = update_rows(opt, w, g, m, v, P["lr"], P["eps"], P["step"], P["beta1"], P["beta2"], P["weight_decay"],
                      P["momentum"], P["eta"], mode)
    want = f64_update(opt, w.astype(np.float64), g.astype(np.float64), None if m is None else m.astype(np.float64),
                      None if v is None else v.astype(np.float64), P, mode)
    tol = (64 + 2 * D) * U
    # error scale of each output: its magnitude plus that of the terms it is formed from (the moments are sums whose
    # terms can cancel)
    scales = {"w": np.abs(want[0]) + np.abs(want[0] - w),
              "m": None if m is None else np.abs(want[1]) + np.abs(m) + np.abs(g),
              "v": None if v is None else np.abs(want[2]) + np.abs(v) + (np.mean(g * g, axis=1) if v.ndim == 1 else g * g)}
    for a, b, what in zip(got, want, ("w", "m", "v")):
        if a is None:
            continue
        assert (np.abs(a - b) <= tol * scales[what] + 1e-30).all(), what


def test_lamb_first_step_moves_each_row_by_lr_times_its_norm():
    """t = 1, wd = 0, zero moments: u = g / (|g| + eps) element-wise, and the step lr |w| / |u| u has norm lr |w|."""
    rng = np.random.default_rng(1)
    w = rng.standard_normal((50, 16)).astype(np.float32)
    g = rng.standard_normal((50, 16)).astype(np.float32)
    z = np.zeros_like(w)
    for opt, v in ((OPT_LAMB, z), (OPT_PARTIAL_ROWWISE_LAMB, np.zeros(50, np.float32))):
        nw, _, _ = update_rows(opt, w, g, z, v, lr=0.1, step=1, weight_decay=0.0)
        step = np.linalg.norm((nw - w).astype(np.float64), axis=1)
        np.testing.assert_allclose(step, 0.1 * np.linalg.norm(w.astype(np.float64), axis=1), rtol=1e-5)


def test_lars_from_zero_momentum_moves_each_row_by_lr_eta_times_its_norm():
    rng = np.random.default_rng(2)
    w = rng.standard_normal((50, 16)).astype(np.float32)
    g = rng.standard_normal((50, 16)).astype(np.float32)
    nw, m, _ = update_rows(OPT_LARS_SGD, w, g, np.zeros_like(w), None, lr=0.5, momentum=0.9, eta=0.001)
    # (w - nw = m up to the rounding of nw: compare the step m itself, not the difference of two close numbers)
    step = np.linalg.norm(m.astype(np.float64), axis=1)
    np.testing.assert_allclose(step, 0.5 * 0.001 * np.linalg.norm(w.astype(np.float64), axis=1), rtol=1e-5)
    np.testing.assert_allclose(w - nw, m, rtol=0, atol=float(np.abs(w).max()) * U)


def test_rowwise_adagrad_l2_is_mode_none_on_the_decayed_gradient():
    """L2: s += mean((g + wd w)^2), w = (1 - mult wd) w - mult g == the plain row-wise update of g + wd w (the classic
    oracle), to rounding."""
    rng = np.random.default_rng(3)
    n, D, wd, lr = 40, 8, 0.05, 0.1
    w = rng.standard_normal((n, D)).astype(np.float32)
    g = rng.standard_normal((n, D)).astype(np.float32)
    s = (rng.random(n) * 0.1).astype(np.float32)
    nw, _, ns = update_rows(O.OPT_ROWWISE_ADAGRAD, w, g, None, s, lr=lr, weight_decay=wd, weight_decay_mode=WD_L2)
    tab, st = w.copy(), s.copy()
    gl = (g + np.float32(wd) * w).astype(np.float32)
    O.fused_update(O.OPT_ROWWISE_ADAGRAD, [tab], [st], [0], [O.POOL_SUM], np.arange(n, dtype=np.int64),
                   np.arange(n + 1, dtype=np.int64), n, gl, lr)
    np.testing.assert_allclose(ns, st, rtol=4 * U * D)
    np.testing.assert_allclose(nw, tab, rtol=0, atol=float(np.max(np.abs(w))) * 16 * U)


def test_degenerate_rows_follow_the_literal_formula():
    """LAMB with u = 0 (zero gradient, zero moments, wd = 0): |w| / |u| = inf, inf * 0 = NaN -> the row is NaN.
    LARS with g = 0 and wd = 0: lr' = x / 0 = inf, m = inf * 0 = NaN.  LARS with w = 0: lr' = 0, w = -momentum m."""
    w = np.ones((1, 4), np.float32)
    z = np.zeros((1, 4), np.float32)
    nw, m, v = update_rows(OPT_LAMB, w, z, z, z, lr=0.1, weight_decay=0.0)
    assert np.isnan(nw).all() and (m == 0).all() and (v == 0).all()
    nw, m, _ = update_rows(OPT_PARTIAL_ROWWISE_LAMB, w, z, z, np.zeros(1, np.float32), lr=0.1, weight_decay=0.0)
    assert np.isnan(nw).all() and (m == 0).all()
    nw, m, _ = update_rows(OPT_LARS_SGD, w, z, z, None, lr=0.1, weight_decay=0.0)
    assert np.isnan(nw).all() and np.isnan(m).all()
    m0 = np.full((1, 4), 0.5, np.float32)
    nw, m, _ = update_rows(OPT_LARS_SGD, z, np.ones((1, 4), np.float32), m0, None, lr=0.1, momentum=0.9)
    np.testing.assert_array_equal(m, np.float32(0.9) * m0)
    np.testing.assert_array_equal(nw, -np.float32(0.9) * m0)


# ---- train_config mapping ---------------------------------------------------------------------------------------------
def _spec(body):
    from torcheasyrec_b200.config import parse_text
    from torcheasyrec_b200.rank_models import sparse_optimizer_from_config

    return sparse_optimizer_from_config(parse_text("train_config { sparse_optimizer { %s } }" % body).train_config)


def test_config_mapping_and_proto_defaults():
    for name, kind in (("lamb", K.OPT_LAMB), ("partial_rowwise_lamb", K.OPT_PARTIAL_ROWWISE_LAMB)):
        s = _spec(f"{name}_optimizer {{ lr: 0.01 }}")
        assert s.kind == kind and abs(s.lr - 0.01) < 1e-9
        assert (s.beta1, s.beta2, s.weight_decay, s.max_gradient) == (0.9, 0.999, 0.0, 0.0)
        s = _spec(f"{name}_optimizer {{ lr: 0.02 beta1: 0.8 beta2: 0.9 weight_decay: 0.01 gradient_clipping: true }}")
        assert abs(s.beta1 - 0.8) < 1e-6 and abs(s.beta2 - 0.9) < 1e-6 and abs(s.weight_decay - 0.01) < 1e-9
        assert s.max_gradient == 1.0                  # proto default max_gradient
    s = _spec("lars_sgd_optimizer { lr: 0.5 }")
    assert s.kind == K.OPT_LARS_SGD and (s.momentum, s.weight_decay, s.eta, s.max_gradient) == (0.9, 0.0, 0.001, 0.0)
    s = _spec("lars_sgd_optimizer { lr: 0.5 momentum: 0.5 weight_decay: 0.001 gradient_clipping: true max_gradient: 2 }")
    assert (s.momentum, s.max_gradient) == (0.5, 2.0) and abs(s.weight_decay - 0.001) < 1e-9
    s = _spec("rowwise_adagrad_optimizer { lr: 0.02 }")
    assert (s.kind, s.weight_decay, s.weight_decay_mode) == (K.OPT_ROWWISE_ADAGRAD, 0.0, K.WD_NONE)
    for mode, want in (("NONE", K.WD_NONE), ("L2", K.WD_L2), ("DECOUPLE", K.WD_DECOUPLE)):
        s = _spec(f"rowwise_adagrad_optimizer {{ lr: 0.02 weight_decay: 0.1 weight_decay_mode: {mode} }}")
        assert s.weight_decay_mode == want and abs(s.weight_decay - 0.1) < 1e-9
    for name in ("adadelta", "rmsprop"):
        with pytest.raises(RuntimeError, match="fbgemm"):
            _spec(f"{name}_optimizer {{ lr: 0.01 }}")


def test_spec_from_name():
    from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec

    assert SparseOptimizerSpec.from_name("LAMB").kind == K.OPT_LAMB
    assert SparseOptimizerSpec.from_name("partial_rowwise_lamb").kind == K.OPT_PARTIAL_ROWWISE_LAMB
    assert SparseOptimizerSpec.from_name("lars_sgd", momentum=0.5).momentum == 0.5


# ---- state layout and checkpoint keys ---------------------------------------------------------------------------------
def _ebc(spec):
    from torcheasyrec_b200.embedding_modules import EmbeddingBagCollection, EmbeddingBagConfig

    m = EmbeddingBagCollection([EmbeddingBagConfig(name="t", num_embeddings=20, embedding_dim=8, feature_names=["f"]),
                                EmbeddingBagConfig(name="u", num_embeddings=7, embedding_dim=4, feature_names=["g"])],
                               device="cpu")
    m.set_optimizer(spec)
    return m


@pytest.mark.parametrize("name,shapes", [
    ("lamb", {"momentum1": (20, 8), "momentum2": (20, 8), "iter": (1,)}),
    ("partial_rowwise_lamb", {"momentum1": (20, 8), "momentum2": (20,), "iter": (1,)}),
    ("lars_sgd", {"momentum1": (20, 8)}),
])
def test_fused_state_keys_and_shapes(name, shapes):
    from torcheasyrec_b200.checkpoint import fused_optimizer_state_dict
    from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec

    m = _ebc(SparseOptimizerSpec.from_name(name, lr=0.1))
    assert m.table_state(1).shape == (7, 4)
    root = torch.nn.Module()
    root.ebc = m
    sd = fused_optimizer_state_dict(root)
    want = {f"state.ebc.embedding_bags.t.weight.t.{k}": v for k, v in shapes.items()}
    got = {k: tuple(v.shape) for k, v in sd.items() if ".t.weight." in k}
    assert got == want


def test_rowwise_adagrad_decay_only_reaches_the_kernel_with_a_mode():
    from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec

    assert _ebc(SparseOptimizerSpec(kind=K.OPT_ROWWISE_ADAGRAD, weight_decay=0.1)).opt_extras() == {}
    ex = _ebc(SparseOptimizerSpec(kind=K.OPT_ROWWISE_ADAGRAD, weight_decay=0.1, weight_decay_mode=K.WD_L2)).opt_extras()
    assert ex == dict(weight_decay=0.1, weight_decay_mode=K.WD_L2, max_gradient=0.0)
    ex = _ebc(SparseOptimizerSpec.from_name("lars_sgd", momentum=0.5, weight_decay=0.01)).opt_extras()
    assert ex == dict(momentum=0.5, eta=0.001, weight_decay=0.01, max_gradient=0.0)
    m = _ebc(SparseOptimizerSpec.from_name("lamb"))
    ex = m.opt_extras()
    assert float(m.opt_step) == 1.0 and ex["state2"] is m.opt_state2 and m.opt_state2.numel() == m.opt_state.numel()


# ---- CPU training steps ------------------------------------------------------------------------------------------------
SPECS = [("lamb", dict(lr=0.01, weight_decay=0.01)), ("partial_rowwise_lamb", dict(lr=0.01, max_gradient=0.5)),
         ("lars_sgd", dict(lr=5.0, momentum=0.9, weight_decay=0.001)),
         ("rowwise_adagrad", dict(lr=0.05, weight_decay=0.01, weight_decay_mode=WD_L2)),
         ("rowwise_adagrad", dict(lr=0.05, weight_decay=0.01, weight_decay_mode=WD_DECOUPLE))]


@pytest.mark.parametrize("name,kw", SPECS, ids=["lamb", "partial_rowwise_lamb", "lars_sgd", "rowwise_adagrad_l2",
                                                "rowwise_adagrad_decouple"])
def test_cpu_pipeline_steps(name, kw):
    """Three DLRM-Criteo steps on small tables with the reference as compute: the loss is finite and moves, and only
    rows the batches touched changed."""
    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec
    from torcheasyrec_b200.engine import Pipeline

    p = Pipeline("dlrm_criteo", device="cpu", max_rows=200, seed=11, capturable=False)
    p.model.set_sparse_optimizer(SparseOptimizerSpec.from_name(name, **kw))
    coll = p.model.sparse_collections()[0]
    w0 = coll.dense_weights().clone()
    losses = []
    with Fn.use_backend(ExtOracleKernels()):
        for i in range(3):
            losses.append(float(p.eager_step(p.synthetic_batch(64, seed=20 + i))))
    assert all(np.isfinite(losses)) and len(set(losses)) == 3
    w1 = coll.dense_weights()
    assert torch.isfinite(w1).all() and not torch.equal(w0, w1)


# ---- DCP round trips (gloo, reference as compute) --------------------------------------------------------------------
def _build(sharding, seed, spec):
    from torcheasyrec_b200.distributed import DenseGradSync, shard_model
    from torcheasyrec_b200.engine import Pipeline
    from torcheasyrec_b200.rank_models import dense_optimizer_from_config

    p = Pipeline("dlrm_criteo", device="cpu", max_rows=300, seed=seed, capturable=False)
    if sharding is not None:
        ref = Pipeline("dlrm_criteo", device="cpu", max_rows=300, seed=seed, capturable=False)
        shard_model(p.model, "cpu", default=sharding, source=ref.model)
        p.dense_optimizer = dense_optimizer_from_config(p.cfg.train_config, p.model.dense_parameters())
        p.grad_sync = DenseGradSync(p.model.dense_parameters())
    p.model.set_sparse_optimizer(spec)
    return p


def _full_states(p):
    """{table.name: full tensor} for the weights and every fused state, whatever the sharding (collective)."""
    from torcheasyrec_b200.checkpoint import _collections, _local_state, _state_names
    from torcheasyrec_b200.distributed import TABLE_WISE, _ShardedBase

    out = {}
    for _, m in _collections(p.model):
        if isinstance(m, _ShardedBase):
            for g in m.groups:
                names = [n for n in _state_names(g.local.optimizer.kind) if n != "iter"]
                for t, c in enumerate(g.configs):
                    out[c.name + ".weight"] = m.gather_full_table(c.name).clone()
                    sh = m.plan[c.name]
                    block = c.num_embeddings if sh.kind == TABLE_WISE else sh.block
                    for nm in names:
                        loc = _local_state(g.local, t, nm)
                        pad = torch.zeros((block,) + tuple(loc.shape[1:]))
                        if loc.shape[0]:
                            pad[:loc.shape[0]] = loc
                        parts = [torch.empty_like(pad) for _ in range(m.world)]
                        dist.all_gather(parts, pad)
                        full = parts[sh.owner] if sh.kind == TABLE_WISE else torch.cat(parts)
                        out[f"{c.name}.{nm}"] = full[:c.num_embeddings].clone()
                    if g.local.opt_step is not None:
                        out[f"{c.name}.iter"] = g.local.opt_step.clone()
        else:
            names = [n for n in _state_names(m.optimizer.kind) if n != "iter"]
            for t, c in enumerate(m._configs):
                out[c.name + ".weight"] = m.table_weight(t).clone()
                for nm in names:
                    out[f"{c.name}.{nm}"] = _local_state(m, t, nm).clone()
                if m.opt_step is not None:
                    out[f"{c.name}.iter"] = m.opt_step.clone()
    return out


def _worker(rank, world, port, tmp, phase, sharding, name, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    try:
        from torcheasyrec_b200 import functional as Fn
        from torcheasyrec_b200.checkpoint import list_checkpoint_keys, restore_model, save_model
        from torcheasyrec_b200.embedding_modules import SparseOptimizerSpec

        spec = SparseOptimizerSpec.from_name(name, lr=0.01, weight_decay=0.01)
        with Fn.use_backend(ExtOracleKernels()):
            if phase == "save":
                p = _build(sharding, 5, spec)
                for i in range(2):
                    p.eager_step(p.synthetic_batch(32, seed=10 + i + 100 * rank))
                save_model(tmp, p.model, p.dense_optimizer)
                full = _full_states(p)
                if rank == 0:
                    torch.save(full, os.path.join(tmp, "expect.pt"))
                    keys = list_checkpoint_keys(tmp)
                    pre = "state.embedding_group.emb_impls.__BASE__.ebc.embedding_bags.cat_0_emb.weight.cat_0_emb."
                    want = {"lars_sgd": {"momentum1"}}.get(name, {"momentum1", "momentum2", "iter"})
                    assert {k[len(pre):] for k in keys if k.startswith(pre)} == want, keys
            else:
                p = _build(sharding, 99, spec)
                p.eager_step(p.synthetic_batch(32, seed=1 + rank))
                restore_model(tmp, p.model, p.dense_optimizer)
                exp = torch.load(os.path.join(tmp, "expect.pt"))
                got = _full_states(p)
                assert set(got) == set(exp)
                for k in exp:
                    assert torch.equal(got[k], exp[k]), k
                p.eager_step(p.synthetic_batch(32, seed=3 + rank))
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _run(world, tmp, phase, sharding, name):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, tmp, phase, sharding, name, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    bad = [(r, m) for r, m in res if m != "ok"]
    assert not bad, "\n".join(f"rank {r}: {m}" for r, m in bad)


@pytest.mark.parametrize("name,save_cfg,load_cfg", [
    ("lamb", (2, "row_wise"), (1, None)),
    ("partial_rowwise_lamb", (2, "row_wise"), (2, "table_wise")),
    ("lars_sgd", (2, "row_wise"), (1, None)),
])
def test_dcp_round_trip(tmp_path, name, save_cfg, load_cfg):
    """Saved by W ranks under one plan, restored under another (W = 2 -> 1, row-wise -> table-wise): weights,
    momentum1 / momentum2 (element-wise or row-wise) and the step counter come back exactly."""
    tmp = str(tmp_path)
    _run(save_cfg[0], tmp, "save", save_cfg[1], name)
    _run(load_cfg[0], tmp, "load", load_cfg[1], name)
