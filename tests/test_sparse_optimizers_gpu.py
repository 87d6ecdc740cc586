"""LAMB, partial row-wise LAMB, LARS-SGD and row-wise Adagrad with L2 / decoupled weight decay in the fused sparse
backward (finish_run_norm, csrc/tzk_bwd.cu) on the H100.

The batches are the exact-row-sum batches of tests/test_fused_bwd_edges.py: every fp32 row sum of the gradient equals
its float64 sum, so the kernel's update is compared with a float64 update of the exact sums and the tolerance only has
to cover the update arithmetic.  Bound, in units u = 2^-24 of the error scale of each output (the sum of the absolute
values of the terms it is formed from, so cancellation inside a moment or in w - step is covered): every fp32 operation
of the update rounds once, powf is within 4 ulp of beta^t, and the longest element-wise chain (LAMB: m, v, two bias
corrections, sqrt, + eps, /, + wd w, * ratio * lr, w -) stays below 20 u; 32 leaves room.  The norms add CH x VEC squares
per lane in sequence and then a log2 G shuffle tree (<= 1 u per addition, relative), halved by the square root; the
LAMB trust ratio and LARS's lr' divide two such norms, so both halves add up: (CH VEC + log2 G + 2) u in all.  At the
widest row (D = 1024: G 32, CH 8, VEC 4) that is 71 u = 4.2e-6 relative."""
import os
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from test_fused_bwd_edges import (DEV, KEY32, U, build_kjt, check_exact, cu, dispatch, make_grad,  # noqa: E402
                                  make_layout, misaligned_grad, row_sums, wide_key_case)

from torcheasyrec_b200.kernels import (OPT_LAMB, OPT_LARS_SGD, OPT_PARTIAL_ROWWISE_LAMB, OPT_ROWWISE_ADAGRAD,  # noqa: E402
                                       POOL_MEAN, POOL_SUM, WD_DECOUPLE, WD_L2)

pytestmark = pytest.mark.gpu

NAMES = {"lamb": (OPT_LAMB, 0), "partial_rowwise_lamb": (OPT_PARTIAL_ROWWISE_LAMB, 0), "lars_sgd": (OPT_LARS_SGD, 0),
         "rowwise_adagrad_l2": (OPT_ROWWISE_ADAGRAD, WD_L2), "rowwise_adagrad_decouple": (OPT_ROWWISE_ADAGRAD, WD_DECOUPLE)}
P = dict(lr=2.0 ** -4, eps=float(np.float32(1e-8)), gs=0.5, beta1=0.5, beta2=0.75, weight_decay=0.125, t=2,
         momentum=0.75, eta=0.25)


def ref_update(opt, mode, g, w, m, v, p):
    """float64 update of one row from its exact gradient sum; returns (w, m, v) and the error scale of each."""
    lr, eps, wd = p["lr"], p["eps"], p["weight_decay"]
    if p.get("max_gradient", 0.0) > 0:
        g = np.clip(g, -p["max_gradient"], p["max_gradient"])
    D = len(g)
    if opt in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB):
        b1, b2, t = p["beta1"], p["beta2"], p["t"]
        nm = b1 * m + (1 - b1) * g
        sm = np.abs(b1 * m) + np.abs((1 - b1) * g)
        if opt == OPT_LAMB:
            nv = b2 * v + (1 - b2) * g * g
            den = np.sqrt(nv / (1 - b2 ** t)) + eps
        else:
            nv = b2 * v + (1 - b2) * np.sum(g * g) / D
            den = np.sqrt(nv / (1 - b2 ** t)) + eps
        mh = (nm / (1 - b1 ** t)) / den
        u = mh + wd * w
        scale = lr * np.linalg.norm(w) / np.linalg.norm(u)
        return (w - scale * u, nm, nv), (np.abs(w) + scale * (np.abs(mh) + np.abs(wd * w)), sm, np.abs(nv))
    if opt == OPT_LARS_SGD:
        wn = np.linalg.norm(w)
        lr_r = lr * p["eta"] * wn / (np.linalg.norm(g) + wd * wn)
        nm = p["momentum"] * m + lr_r * (g + wd * w)
        sm = np.abs(p["momentum"] * m) + lr_r * (np.abs(g) + np.abs(wd * w))
        return (w - nm, nm, v), (np.abs(w) + sm, sm, None)
    gl = g + wd * w if mode == WD_L2 else g
    s = v + np.sum(gl * gl) / D
    mult = lr / (np.sqrt(s) + eps)
    keep = 1 - mult * wd if mode == WD_L2 else 1 - lr * wd
    return (keep * w - mult * g, m, s), (np.abs(keep * w) + np.abs(mult * g), None, abs(s))


def budget(dim, vec):
    g, ch = dispatch(dim, vec)
    return (32 + ch * vec + int(np.log2(g)) + 2) * U


def run(kernels, opt, mode, lay, kjt, grad, p, seed=0, grad_t=None, f16=False, state_keys=None):
    """One fused_bwd call on random weights and states; returns inputs and outputs as numpy arrays."""
    rng = np.random.default_rng(seed)
    dlay = lay.to(DEV)
    w0 = (rng.standard_normal(lay.arena_elems) * 0.25).astype(np.float16 if f16 else np.float32)
    n_rw = state_keys or lay.total_keys
    m0 = v0 = None
    ex = dict(weight_decay=p["weight_decay"])
    if opt == OPT_ROWWISE_ADAGRAD:
        v0 = (rng.random(n_rw) * 0.01).astype(np.float32)
        state = cu(v0)
        ex["weight_decay_mode"] = mode
    else:
        m0 = (rng.standard_normal(lay.arena_elems) * 0.01).astype(np.float32)
        state = cu(m0)
        if opt == OPT_LAMB:
            v0 = (rng.random(lay.arena_elems) * 0.01).astype(np.float32)
        elif opt == OPT_PARTIAL_ROWWISE_LAMB:
            v0 = (rng.random(n_rw) * 0.01).astype(np.float32)
    if opt in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB):
        ex.update(state2=cu(v0), step=torch.full((), float(p["t"]), device=DEV), beta1=p["beta1"], beta2=p["beta2"])
    if opt == OPT_LARS_SGD:
        ex.update(momentum=p["momentum"], eta=p["eta"])
    if p.get("max_gradient", 0.0) > 0:
        ex["max_gradient"] = p["max_gradient"]
    arena = cu(w0)
    kernels.fused_bwd(opt, kjt.pooled, cu(grad) if grad_t is None else grad_t, arena, state, dlay, cu(kjt.ids),
                      cu(kjt.offsets), kjt.B, p["lr"], p["eps"], p["gs"], **ex)
    torch.cuda.synchronize()
    m = state.cpu().numpy() if opt != OPT_ROWWISE_ADAGRAD else None
    v = (state if opt == OPT_ROWWISE_ADAGRAD else ex.get("state2", state)).cpu().numpy() if v0 is not None else None
    return dict(w0=w0, m0=m0, v0=v0, w=arena.cpu().numpy(), m=m, v=v)


def check(opt, mode, lay, kjt, grad, r, p, vec, f16=False):
    uk, S = row_sums(lay, kjt, grad, p["gs"])
    B = budget(lay.max_dim, vec)
    w0 = r["w0"].astype(np.float64)
    want_w, tol_w = w0.copy(), np.zeros(len(w0))
    rowwise = opt in (OPT_PARTIAL_ROWWISE_LAMB, OPT_ROWWISE_ADAGRAD)
    want_m = None if r["m0"] is None else r["m0"].astype(np.float64)
    tol_m = None if r["m0"] is None else np.zeros(len(want_m))
    want_v = None if r["v0"] is None else r["v0"].astype(np.float64)
    tol_v = None if r["v0"] is None else np.zeros(len(want_v))
    done = set()
    for f in range(lay.num_features):
        kb, d = lay.key_base[f], lay.dim[f]
        if lay.rows[f] == 0 or (kb, lay.w_off[f]) in done:
            continue
        done.add((kb, lay.w_off[f]))
        for i in np.flatnonzero((uk >= kb) & (uk < kb + lay.rows[f])):
            k = int(uk[i])
            sl = slice(lay.w_off[f] + (k - kb) * d, lay.w_off[f] + (k - kb + 1) * d)
            m = None if want_m is None else r["m0"][sl].astype(np.float64)
            v = None if want_v is None else (float(r["v0"][k]) if rowwise else r["v0"][sl].astype(np.float64))
            (nw, nm, nv), (sw, sm, sv) = ref_update(opt, mode, S[i, :d], w0[sl], m, v, p)
            want_w[sl], tol_w[sl] = nw, B * sw
            if f16:
                tol_w[sl] += 0.5 * np.spacing(np.abs(nw).astype(np.float16)).astype(np.float64)
            if want_m is not None:
                want_m[sl], tol_m[sl] = nm, B * sm
            if want_v is not None:
                if rowwise:
                    want_v[k], tol_v[k] = nv, B * sv
                else:
                    want_v[sl], tol_v[sl] = nv, B * sv
    err = np.abs(r["w"].astype(np.float64) - want_w)
    assert (err <= tol_w).all(), f"weights: max err/tol {np.max(err / np.maximum(tol_w, 1e-300)):.3g}"
    if want_m is not None:
        assert (np.abs(r["m"] - want_m) <= tol_m).all(), "momentum1"
    if want_v is not None:
        assert (np.abs(r["v"] - want_v) <= tol_v).all(), "momentum2 / row-wise state"


def case(seed, dims, pooled=True, pool=POOL_MEAN):
    """One table per dim, two features each; runs of 1, 3, 32, 33, 257 and 300 positions (the last two take the
    long-run chunk CTAs, 300 > 256 the multi-chunk combine) next to random short runs."""
    rng = np.random.default_rng(seed)
    lay = make_layout([(48, d) for d in dims], [t for t in range(len(dims)) for _ in range(2)], pool)
    ks, cs = [], []
    for t in range(len(dims)):
        c = rng.integers(0, 5, 48)
        c[[3, 7, 11, 19, 23, 40]] = [1, 3, 32, 33, 257, 300]
        ks.append(lay.key_base[2 * t] + np.arange(48)); cs.append(c)
    kjt = build_kjt(rng, lay, np.concatenate(ks), np.concatenate(cs), pooled=pooled)
    return lay, kjt, make_grad(rng, lay, kjt)


def _params():
    out = []
    for name in NAMES:
        for dims, vec, layout in [((16,), 4, "mean"), ((16,), 4, "sum"), ((16,), 4, "sequence"), ((4,), 4, "mean"),
                                  ((3,), 1, "mean"), ((68,), 4, "mean"), ((128,), 4, "sequence"), ((260,), 4, "mean"),
                                  ((1, 65), 1, "mean"), ((64,), 1, "mean"), ((1024,), 4, "mean")]:
            g, ch = dispatch(max(dims), vec)
            tag = "x".join(map(str, dims))
            out.append(pytest.param(name, dims, vec, layout, id=f"{name}-d{tag}-G{g}-V{vec}-CH{ch}-{layout}"))
    return out


@pytest.mark.parametrize("name,dims,vec,layout", _params())
def test_kernel_matches_float64_update(kernels, monkeypatch, name, dims, vec, layout):
    """Every (G, VEC, CH) of the general path (VEC 1 from odd dims or from a grad_out column slice with an odd ld_grad),
    pooled MEAN / SUM and the sequence layout, hot rows on the long-run chunk path.  TZK_BWD_TILE=1 is set: these
    optimizers refuse the tile path and take the general one."""
    monkeypatch.setenv("TZK_BWD_TILE", "1")
    opt, mode = NAMES[name]
    pooled = layout != "sequence"
    lay, kjt, grad = case(zlib.crc32(f"norm{name}{dims}{layout}".encode()), dims, pooled,
                          POOL_SUM if layout == "sum" else POOL_MEAN)
    check_exact(lay, kjt, grad, P["gs"])
    natural = 4 if all(d % 4 == 0 for d in dims) else 1
    grad_t = misaligned_grad(grad) if vec < natural else None
    r = run(kernels, opt, mode, lay, kjt, grad, P, seed=max(dims), grad_t=grad_t)
    check(opt, mode, lay, kjt, grad, r, P, vec)
    assert budget(lay.max_dim, vec) <= 1e-5          # the derived bound, relative to each output's error scale


@pytest.mark.parametrize("name", list(NAMES))
@pytest.mark.parametrize("dims", [(16,), (260,)])
def test_clipping(kernels, name, dims):
    opt, mode = NAMES[name]
    lay, kjt, grad = case(zlib.crc32(f"clip{name}{dims}".encode()), dims)
    p = dict(P, max_gradient=0.25)
    r = run(kernels, opt, mode, lay, kjt, grad, p, seed=5)
    check(opt, mode, lay, kjt, grad, r, p, 4)


@pytest.mark.parametrize("name", list(NAMES))
@pytest.mark.parametrize("dims", [(16,), (3,), (260,)])
def test_fp16_tables(kernels, name, dims):
    """FP16 arena: the row is widened, updated in fp32 (norms included) and rounded to nearest: within half an ulp of
    the stored half plus the fp32 bound."""
    opt, mode = NAMES[name]
    lay, kjt, grad = case(zlib.crc32(f"f16{name}{dims}".encode()), dims)
    r = run(kernels, opt, mode, lay, kjt, grad, P, seed=6, f16=True)
    check(opt, mode, lay, kjt, grad, r, P, 4 if dims[0] % 4 == 0 else 1, f16=True)


@pytest.mark.parametrize("name", ["lamb", "lars_sgd"])
def test_key_base_above_2_32(kernels, name):
    """uint64 keys, a table whose key base is above 2^32 (element-wise states only: a row-wise state indexed by key
    would need 2^32 entries here)."""
    opt, mode = NAMES[name]
    lay, kjt, grad = wide_key_case("high_base")
    r = run(kernels, opt, mode, lay, kjt, grad, P)
    check(opt, mode, lay, kjt, grad, r, P, 4)


@pytest.mark.parametrize("name", ["partial_rowwise_lamb", "rowwise_adagrad_l2"])
def test_rowwise_state_on_uint64_keys(kernels, name):
    opt, mode = NAMES[name]
    lay = make_layout([(KEY32 + 7, 16)], [0, 0], POOL_MEAN, stored=[64])
    rng = np.random.default_rng(3)
    counts = rng.integers(0, 5, 64)
    counts[[2, 9]] = [33, 600]
    kjt = build_kjt(rng, lay, np.arange(64), counts)
    grad = make_grad(rng, lay, kjt)
    r = run(kernels, opt, mode, lay, kjt, grad, P, state_keys=64)
    check(opt, mode, lay, kjt, grad, r, P, 4)


def test_degenerate_rows(kernels):
    """A row whose gradient contributions cancel exactly (g = 0), with zero moments and wd = 0: LAMB's |u| = 0 and
    LARS's |g| + wd |w| = 0 make the row NaN, as the literal formula does (and tests/sparse_optim_ref.py); a zero row
    under LARS moves by -momentum m.  Other rows are finite."""
    lay = make_layout([(8, 4)], [0], POOL_SUM)
    dlay = lay.to(DEV)
    ids = cu(np.array([0, 0, 1, 2], np.int64))
    offs = cu(np.array([0, 1, 2, 3, 4], np.int64))
    grad = cu(np.array([[0.5] * 4, [-0.5] * 4, [0.25] * 4, [0.125] * 4], np.float32))
    for opt in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB, OPT_LARS_SGD):
        w = torch.ones(lay.arena_elems, device=DEV)
        w[8:12] = 0.0                                          # row 2: a zero row
        m = torch.zeros(lay.arena_elems, device=DEV)
        m[8:12] = 0.5
        ex = dict(weight_decay=0.0)
        if opt == OPT_LARS_SGD:
            ex.update(momentum=0.75, eta=0.5)
        else:
            ex.update(state2=torch.zeros(lay.arena_elems if opt == OPT_LAMB else lay.total_keys, device=DEV),
                      step=torch.ones((), device=DEV))
        kernels.fused_bwd(opt, True, grad, w, m, dlay, ids, offs, 4, 0.1, 1e-8, 1.0, **ex)
        wn = w.cpu().numpy()
        assert np.isnan(wn[0:4]).all(), opt
        assert np.isfinite(wn[4:]).all(), opt
        if opt == OPT_LARS_SGD:
            np.testing.assert_array_equal(wn[8:12], np.full(4, -0.375, np.float32))
            assert np.isnan(m.cpu().numpy()[0:4]).all()


@pytest.mark.parametrize("name", ["lamb", "partial_rowwise_lamb", "lars_sgd"])
def test_graph_replay_matches_eager_bit_for_bit(kernels, name):
    """Five steps, each `step += 1` on the device and one fused_bwd: eagerly, and as one captured CUDA graph replayed
    five times — the same bits (the bias correction reads the device step counter)."""
    opt, mode = NAMES[name]
    lay, kjt, grad = case(77, (16, 64))
    dlay = lay.to(DEV)
    ids, offs, g = cu(kjt.ids), cu(kjt.offsets), cu(grad)
    rng = np.random.default_rng(8)
    w0 = cu((rng.standard_normal(lay.arena_elems) * 0.25).astype(np.float32))

    def fresh():
        st = dict(w=w0.clone(), m=torch.zeros(lay.arena_elems, device=DEV), step=torch.zeros((), device=DEV))
        st["v"] = torch.zeros(lay.arena_elems if opt == OPT_LAMB else lay.total_keys, device=DEV)
        return st

    def one(st):
        st["step"].add_(1.0)
        ex = dict(weight_decay=0.01)
        if opt == OPT_LARS_SGD:
            ex.update(momentum=0.9, eta=0.01)
        else:
            ex.update(state2=st["v"], step=st["step"])
        kernels.fused_bwd(opt, True, g, st["w"], st["m"], dlay, ids, offs, kjt.B, 0.05, 1e-8, 0.5, **ex)

    eager = fresh()
    for _ in range(5):
        one(eager)
    graphed = fresh()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):             # warm-up (workspace allocation) on a scratch copy
        one(fresh())
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one(graphed)
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert float(graphed["step"]) == 5.0
    for k in ("w", "m", "v"):
        assert torch.equal(eager[k], graphed[k]), k


def _peer_helpers():
    import test_peer_gpu as PG

    return PG


@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("name", ["lamb", "lars_sgd"])
def test_peer_step_on_one_gpu(kernels, W, name):
    """The peer-memory sharded step (W virtual ranks on one GPU, as tests/test_peer_gpu.py) with LAMB / LARS: the
    gathered shards after two steps match the unsharded collection stepped on the concatenated batch."""
    PG = _peer_helpers()
    M = PG._helpers()
    from torcheasyrec_b200 import peer_exchange
    from torcheasyrec_b200.distributed import TABLE_WISE, make_plan
    from torcheasyrec_b200.embedding_modules import EmbeddingBagCollection, SparseOptimizerSpec

    torch.manual_seed(0)
    B = 257
    rng = np.random.default_rng(W * 7)
    cfgs = M._pooled_configs()
    D = 16
    plan = make_plan(cfgs, W, "row_wise", {"t_tw": [TABLE_WISE], "t_tiny": [TABLE_WISE]})
    spec = SparseOptimizerSpec.from_name(name, lr=0.05 if name == "lamb" else 5.0, weight_decay=0.01)
    full = EmbeddingBagCollection(cfgs, device="cuda")
    full.set_optimizer(spec)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    groups = PG._seed_groups(cfgs, plan, W, True, full, spec, 2.5)
    batches = [M._bags(rng, F, B, feat_rows, False) for _ in range(W)]
    ids, offs = [b[0].cuda() for b in batches], [b[1].cuda() for b in batches]
    grads = [torch.from_numpy(rng.standard_normal((B, F * D)).astype(np.float32)).cuda() for _ in range(W)]
    registry = {}
    budget_ = [B] * F

    def body(r, tbar):
        torch.cuda.set_device(0)

        class St(M._sim_mixin(registry, tbar, "gpu", "cuda"), peer_exchange.PeerState):
            pass

        st = St(groups[r], plan, None, B, budget_)
        for _ in range(2):
            st.gather(ids[r], offs[r])
            st.prep(ids[r], offs[r])
            st.backward(grads[r], offs[r])
            torch.cuda.synchronize()

    M._run_ranks(W, body)
    assert all(int(g.overflow.item()) == 0 for g in groups)
    cat = M._cat_key_major([i.cpu() for i in ids], [o.cpu() for o in offs], F, B, W)
    cat_ids, cat_off = cat[0].cuda(), cat[1].cuda()
    cat_grad = torch.cat(grads) / W
    for _ in range(2):
        kernels.fused_bwd(spec.kind, True, cat_grad, full.weights.data, full.opt_state, full.layout, cat_ids, cat_off,
                          B * W, spec.lr, spec.eps, 1.0, **full.opt_extras())
    for t, c in enumerate(cfgs):
        torch.testing.assert_close(PG._gathered(groups, plan, cfgs, full, t), full.table_weight(t), rtol=5e-5, atol=1e-6,
                                   msg=lambda m, c=c: f"{c.name}: {m}")


def test_graphed_train_step_with_lamb():
    """GraphedTrainStep on DLRM-Criteo with train_config.sparse_optimizer { lamb_optimizer }: replays run and the loss
    stays finite; the step counter advances once per replay."""
    from torcheasyrec_b200.config import parse_text
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline
    from torcheasyrec_b200.rank_models import sparse_optimizer_from_config

    spec = sparse_optimizer_from_config(parse_text(
        "train_config { sparse_optimizer { lamb_optimizer { lr: 0.01 weight_decay: 0.001 } } }").train_config)
    p = Pipeline("dlrm_criteo", device="cuda:0", max_rows=5000, seed=3)
    p.model.set_sparse_optimizer(spec)
    batches = [p.synthetic_batch(1024, seed=40 + i) for i in range(3)]
    step = GraphedTrainStep(p, batches[0], warmup=3)
    n0 = float(p.model.sparse_collections()[0].opt_step)
    losses = []
    for b in batches:
        step.load(b.pin_memory())
        losses.append(float(step.replay()))
    assert all(np.isfinite(losses)), losses
    assert float(p.model.sparse_collections()[0].opt_step) == n0 + 3
