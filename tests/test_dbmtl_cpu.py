"""DBMTL and the JRC loss on the CPU: the float64 restatement (tests/dbmtl_ref.py) and functional.torch_jrc_loss pinned
to the reference's own JRCLoss (tests/golden/ref_dbmtl.npz, made by tests/golden/make_dbmtl_golden.py), the SOURCE of the
fused loss (csrc/tzk_jrc.cuh) run on the host through tests/native/cuda_cpu_shim.h against float64, and the model:
reference parameter names and widths, two-class heads, the NaN rules, refusals, the example configs trained with the
fused loss path (checker backend) and evaluation."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import dbmtl_ref as R  # noqa: E402
from metric_oracle_backend import MetricOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.example_configs import GENERATORS  # noqa: E402
from torcheasyrec_b200.features import create_features  # noqa: E402
from torcheasyrec_b200.rank_models import JRCLoss, create_model  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ref_dbmtl.npz"))
NATIVE = os.path.join(HERE, "native")
REF_EXAMPLES = os.path.join(HERE, "golden", "ref_examples")


def _close(got, want, r, name=""):
    """|got - want| <= r (|want| + max(1, max |want|)), NaN where want is NaN."""
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, float(np.nanmax(np.abs(want))) if want.size else 1.0), err_msg=name)


def _golden():
    for tag in R.CASES:
        logits, y, s, w = R.seeded_case(tag)
        for alpha in R.ALPHAS:
            for red in ("mean", "none"):
                if red == "mean" and w is not None:
                    continue
                ww = None if red == "mean" else (w if w is not None else np.ones(len(y)))
                yield f"{tag}_{alpha}_{red}", logits, y, s, ww, alpha


GOLDEN = list(_golden())
IDS = [g[0] for g in GOLDEN]


# ---- the restatements, pinned to the reference's JRCLoss ---------------------------------------------------------------
@pytest.mark.parametrize("case", GOLDEN, ids=IDS)
def test_restatement_matches_reference_jrc(case):
    key, logits, y, s, w, alpha = case
    loss, grad = R.jrc(logits, y, s, alpha, w)
    tol = 1e-6 if w is None else 2e-6          # "none" was run by the reference in float32
    _close(loss, GOLD[key + "_loss"], tol, "loss")
    _close(grad, GOLD[key + "_dlogits"], tol, "dlogits")


@pytest.mark.parametrize("case", GOLDEN, ids=IDS)
def test_torch_jrc_matches_reference_jrc(case):
    """functional.jrc_loss off the fused path (CPU tensors, no test backend): the O(B) torch formulation."""
    key, logits, y, s, w, alpha = case
    lg = torch.tensor(logits, dtype=torch.float64, requires_grad=True)
    loss = Fn.jrc_loss(lg, torch.tensor(y), torch.tensor(s), alpha, None if w is None else torch.tensor(w))
    loss.backward()
    _close(loss.item(), GOLD[key + "_loss"], 2e-5, "loss")
    _close(lg.grad.numpy(), GOLD[key + "_dlogits"], 2e-5, "dlogits")


def test_jrc_module_reductions():
    logits, y, s, _ = R.seeded_case("mixed")
    lg, yt, st = torch.tensor(logits).float(), torch.tensor(y).long(), torch.tensor(s)
    per = JRCLoss(0.3, "none")(lg, yt, st)
    assert per.shape == (len(y),)
    _close(per.mean().item(), GOLD["mixed_0.3_none_loss"], 2e-5)
    _close(JRCLoss(0.3)(lg, yt, st).item(), GOLD["mixed_0.3_mean_loss"], 2e-5)
    with pytest.raises(ValueError):
        JRCLoss(0.5, "sum")


def test_single_class_batch_is_nan_with_finite_gradient():
    """Mean mode: no positive (or no negative) gives the reference's NaN loss; the gradient is the CE term plus the
    present class's term.  The per-sample (none) reduction has no NaN."""
    for tag in ("all_negative", "all_positive"):
        logits, y, s, _ = R.seeded_case(tag)
        lg = torch.tensor(logits, requires_grad=True)
        loss = Fn.jrc_loss(lg, torch.tensor(y), torch.tensor(s), 0.5)
        loss.backward()
        assert torch.isnan(loss)
        assert torch.isfinite(lg.grad).all()
        _close(lg.grad.numpy(), GOLD[f"{tag}_0.5_mean_dlogits"], 2e-5)
        assert torch.isfinite(Fn.torch_jrc_loss(lg.detach(), torch.tensor(y), torch.tensor(s), 0.5, "none")).all()


def test_label_outside_01_gives_nan():
    """Where the reference raises inside CrossEntropyLoss, the loss is NaN (no assert, no host read on the fused path)."""
    logits, y, s, _ = R.seeded_case("mixed")
    y = y.copy()
    y[3] = 2.0
    loss = Fn.jrc_loss(torch.tensor(logits), torch.tensor(y), torch.tensor(s), 0.5)
    assert torch.isnan(loss)


# ---- the kernel source on the host -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libjrc_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "jrc_standalone.cu"), "-shared", "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    P = ctypes.c_void_p
    L.jrc_loss.argtypes = [P, ctypes.c_int64, P, P, P, ctypes.c_int64, ctypes.c_float, P, P]
    L.jrc_loss.restype = ctypes.c_int
    return L


def _run_kernel(L, logits, y, s, w, alpha):
    lg = np.ascontiguousarray(logits, np.float32)
    yy = np.ascontiguousarray(y, np.float32)
    ss = np.ascontiguousarray(s, np.int64)
    ww = None if w is None else np.ascontiguousarray(w, np.float32)
    B = len(yy)
    loss = np.full(1, -1.0, np.float32)
    d = np.full((B, 2), np.nan, np.float32)
    ptr = lambda a: None if a is None else a.ctypes.data
    assert L.jrc_loss(ptr(lg), 2, ptr(yy), ptr(ss), ptr(ww), B, alpha, ptr(loss), ptr(d)) == 0
    return loss[0], d


def _kernel_cases():
    yield from GOLDEN
    rng = np.random.default_rng(5)
    B = 700                                     # sessions across the 256-position chunks of the kernel
    lg = rng.normal(0, 3, (B, 2))
    y = (rng.random(B) < 0.3).astype(np.float64)
    yield "one_session_700", lg, y, np.full(B, 4, np.int64), None, 0.5
    s = np.sort(rng.integers(0, 6, B)) * 1000 + 7
    yield "six_sessions_700", lg, y, rng.permutation(s), rng.uniform(0, 2, B), 0.3
    lens = [255, 1, 257, 187]                   # runs that end exactly at and just past a chunk boundary
    s = np.concatenate([np.full(n, k, np.int64) for k, n in enumerate(lens)])
    yield "boundaries_700", lg, y, s, None, 0.5
    yield "B1_pos", np.array([[0.3, -1.2]]), np.array([1.0]), np.array([9], np.int64), None, 0.5
    yield "B1_weighted", np.array([[0.3, -1.2]]), np.array([0.0]), np.array([9], np.int64), np.array([1.5]), 0.5


KCASES = list(_kernel_cases())


@pytest.mark.parametrize("case", KCASES, ids=[c[0] for c in KCASES])
def test_kernel_source_matches_float64(kern, case):
    key, logits, y, s, w, alpha = case
    want_loss, want_d = R.jrc(logits, y, s, alpha, w)
    loss, d = _run_kernel(kern, logits, y, s, w, alpha)
    _close(loss, want_loss, 1e-5, "loss")
    assert np.isfinite(d).all()
    np.testing.assert_allclose(d, want_d, rtol=0, atol=1e-5 * max(np.abs(want_d).max(), 1e-30))
    loss2, d2 = _run_kernel(kern, logits, y, s, w, alpha)
    assert np.array_equal(d, d2) and (np.isnan(loss) and np.isnan(loss2) or loss.tobytes() == loss2.tobytes())


def test_kernel_source_empty_batch_and_bad_label(kern):
    loss, d = _run_kernel(kern, np.zeros((0, 2)), np.zeros(0), np.zeros(0, np.int64), None, 0.5)
    assert np.isnan(loss) and d.shape == (0, 2)
    logits, y, s, _ = R.seeded_case("mixed")
    y = y.copy()
    y[5] = 3.0
    loss, d = _run_kernel(kern, logits, y, s, None, 0.5)
    assert np.isnan(loss)
    i = 5
    assert np.isnan(d[i]).all() and np.isfinite(np.delete(d, i, axis=0)).all()


# ---- the model --------------------------------------------------------------------------------------------------------
class JrcOracleKernels(MetricOracleKernels):
    """The CPU checker backend with the JRC loss: the float64 restatement rounded to fp32, with the CUDA backend's
    signature, counting its calls."""

    def __init__(self) -> None:
        super().__init__(False)
        self.jrc_calls = 0

    def jrc_loss(self, logits, labels, session_ids, weights, alpha, key_bits=64):
        self.jrc_calls += 1
        assert logits.dtype == torch.float32 and labels.dtype == torch.float32 and session_ids.dtype == torch.int64
        assert int(session_ids.max()) < (1 << key_bits) if session_ids.numel() else True
        loss, d = R.jrc(logits.detach().double().numpy(), labels.numpy(), session_ids.numpy(), alpha,
                        None if weights is None else weights.double().numpy())
        return torch.tensor(loss, dtype=torch.float32), torch.from_numpy(d).float()


def _model(text):
    """The config's model on the CPU, tables capped at 1000 rows."""
    text = re.sub(r"num_buckets: (\d+)", lambda m: f"num_buckets: {min(int(m.group(1)), 1000)}", text)
    cfg = parse_text(text)
    feats = create_features(list(cfg.feature_configs), fg_mode=cfg.data_config.fg_mode)
    return create_model(cfg.model_config, feats, list(cfg.data_config.label_fields),
                        device=torch.device("cpu"))


def test_dbmtl_parameter_names_and_widths():
    """dbmtl.py's module names and its input-width rules, including a relation tower without an MLP (counted with the
    tower input's width) and a relation chain of three towers."""
    text = GENERATORS["dbmtl_taobao"]()
    text = text.replace('            relation_tower_names: "ctr"\n',
                        '            relation_tower_names: "ctr"\n            relation_tower_names: "x"\n')
    text = text.replace("    dbmtl {\n", "    dbmtl {\n        task_towers {\n            tower_name: \"x\"\n"
                        "            label_name: \"clk\"\n            losses {\n                binary_cross_entropy {}\n"
                        "            }\n        }\n")
    m = _model(text)
    names = [k for k, _ in m.named_parameters() if not k.startswith("embedding_group")]
    assert names[:2] == ["bottom_mlp.mlp.0.perceptron.0.weight", "bottom_mlp.mlp.0.perceptron.0.bias"]
    assert "task_mlps.ctr.mlp.2.perceptron.0.weight" in names and "relation_mlps.cvr.mlp.0.perceptron.0.weight" in names
    assert "task_mlps.x.mlp.0.perceptron.0.weight" not in names
    assert m.relation_mlps["cvr"].mlp[0].perceptron[0].weight.shape == (64, 64 + 64 + 512)
    assert [tuple(o.weight.shape) for o in m.task_outputs] == [(1, 512), (1, 64), (1, 64)]


def test_refusals():
    base = GENERATORS["dbmtl_taobao"]()
    with pytest.raises(NotImplementedError, match="softmax_cross_entropy"):
        _model(base.replace("binary_cross_entropy {}", "softmax_cross_entropy {}", 1))
    with pytest.raises(NotImplementedError, match="sample_weight_name"):
        _model(base.replace('label_name: "clk"\n', 'label_name: "clk"\n            sample_weight_name: "w"\n', 1))
    with pytest.raises(NotImplementedError, match="pareto"):
        _model(base.replace("model_config {\n", "model_config {\n    use_pareto_loss_weight: true\n"))
    with pytest.raises(AssertionError, match="num_class must be 2"):
        _model(GENERATORS["dbmtl_taobao_jrc"]().replace("num_class: 2\n", "", 1))
    with pytest.raises(NotImplementedError, match="jrc_loss"):    # MMoE's towers keep BCE only
        _model(GENERATORS["mmoe_taobao"]().replace("binary_cross_entropy {}",
                                                   'jrc_loss { session_name: "user_id" }', 1))


@pytest.mark.parametrize("name", ["dbmtl_taobao", "dbmtl_taobao_jrc"])
def test_reference_example_trains_with_fused_loss(name):
    """The reference's file as stored, stepped on the CPU with the checker backend: finite falling losses; the JRC
    towers go through the fused loss path (one call per tower per step) with the session ids of user_id."""
    pipe =Pipeline(os.path.join(REF_EXAMPLES, name + ".config"), device="cpu", max_rows=200, seed=3)
    batch = pipe.synthetic_batch(48, seed=1)
    be = JrcOracleKernels()
    with Fn.use_backend(be):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all() and l1 < l0
    assert be.jrc_calls == (4 if name.endswith("jrc") else 0)


def test_jrc_predictions_loss_and_weighting():
    m = _model(GENERATORS["dbmtl_taobao_jrc"]())
    feats = m._features
    from torcheasyrec_b200.batch import synthetic_batch

    batch = synthetic_batch(feats, 32, ["clk", "buy"], seed=2)
    with Fn.use_backend(JrcOracleKernels()):
        preds = m.predict(batch)
        assert preds["logits_ctr"].shape == (32, 2) and preds["probs1_ctr"].shape == (32,)
        torch.testing.assert_close(preds["probs_ctr"], torch.softmax(preds["logits_ctr"], 1))
        losses = m.loss(preds, batch)
    assert set(losses) == {"jrc_loss_ctr", "jrc_loss_cvr"}
    sid = m._session_ids(batch, "user_id")
    from torcheasyrec_b200.features import BASE_DATA_GROUP

    with Fn.use_backend(JrcOracleKernels()):
        want_sid = batch.sparse_features[BASE_DATA_GROUP].to_dict()["user_id"].to_padded_dense(1)[:, 0]
    assert torch.equal(sid, want_sid)
    want = Fn.torch_jrc_loss(preds["logits_ctr"], batch.labels["clk"], sid, 0.5)
    _close(losses["jrc_loss_ctr"].item(), want.item(), 1e-5)
    # a tower with `weight` takes the per-sample reduction weighted by div_no_nan(v, mean v) * weight
    mw = _model(GENERATORS["dbmtl_taobao_jrc"]().replace('label_name: "clk"\n',
                                                        'label_name: "clk"\n            weight: 0.5\n', 1))
    mw.load_state_dict(m.state_dict())
    with Fn.use_backend(JrcOracleKernels()):
        lw = mw.loss(mw.predict(batch), batch)["jrc_loss_ctr"]
    per = Fn.torch_jrc_loss(preds["logits_ctr"], batch.labels["clk"], sid, 0.5, "none")
    _close(lw.item(), (per * 0.5).mean().item(), 1e-5)


def test_evaluate_reports_auc_and_jrc_loss():
    m = _model(GENERATORS["dbmtl_taobao_jrc"]())
    feats = m._features
    from torcheasyrec_b200.batch import synthetic_batch

    m.eval()
    be = JrcOracleKernels()
    with Fn.use_backend(be):
        m.init_metric(device=torch.device("cpu"))
        for seed in range(2):
            batch = synthetic_batch(feats, 40, ["clk", "buy"], seed=seed)
            with torch.no_grad():
                p = m.predict(batch)
                m.update_metric(p, batch, m.loss(p, batch))
        out = m.compute_metric()
    assert set(out) == {"auc_ctr", "auc_cvr", "jrc_loss_ctr", "jrc_loss_cvr"}


def test_synthetic_sessions_only_for_jrc_configs():
    """A jrc_loss config draws its session feature over ceil(B / 8) ids; every other config's batch is unchanged."""
    from torcheasyrec_b200.features import BASE_DATA_GROUP

    jrc = Pipeline(os.path.join(REF_EXAMPLES, "dbmtl_taobao_jrc.config"), device="cpu", max_rows=200, seed=3)
    b = jrc.synthetic_batch(64, seed=1)
    sid = b.sparse_features[BASE_DATA_GROUP].to_dict()["user_id"].values()
    assert int(sid.max()) < 8 and len(torch.unique(sid)) > 1
    plain = Pipeline(os.path.join(REF_EXAMPLES, "dbmtl_taobao.config"), device="cpu", max_rows=200, seed=3)
    from torcheasyrec_b200.batch import synthetic_batch

    ref = synthetic_batch(plain.features, 64, plain.labels, seed=1)
    got = plain.synthetic_batch(64, seed=1)
    assert torch.equal(got.sparse_features[BASE_DATA_GROUP].values(), ref.sparse_features[BASE_DATA_GROUP].values())


# ---- this repo's DBMTL against the reference's own (tests/golden/ref_dbmtl.npz model cases) -------------------------
@pytest.mark.parametrize("tag", list(R.MODEL_CASES))
def test_dbmtl_matches_reference_model(tag):
    """State-dict keys, tower outputs, the input gradient and every parameter gradient of this repo's DBMTL, built from
    the case as a config and fed the seeded group input in place of the embedding lookup, against the reference's."""
    from oracle_backend import OracleKernels

    m = _model(R.model_config_text(tag))
    pre = f"model_{tag}_"
    keys = [k for k in m.state_dict() if not k.startswith("embedding_group")]
    assert keys == list(GOLD[pre + "keys"])
    m.load_state_dict({k: torch.from_numpy(GOLD[pre + "sd__" + k]).float() for k in keys}, strict=False)
    x = torch.from_numpy(R.seeded_state(tag, {})[1]).float().requires_grad_(True)
    m.build_input = lambda batch: {"all": x}
    dys = R.seeded_state(tag, {})[2]
    with Fn.use_backend(OracleKernels()):
        preds = m.predict(None)
        outs = {t: preds[f"logits_{t}"] for t in dys}
        outs = {t: (o if o.dim() == 2 else o.unsqueeze(1)) for t, o in outs.items()}
        torch.autograd.backward(list(outs.values()), [torch.from_numpy(dys[t]).float() for t in outs])
    for t, o in outs.items():
        _close(o.detach().numpy(), GOLD[pre + "out__" + t], 2e-5, t)
    _close(x.grad.numpy(), GOLD[pre + "dx"], 2e-5, "dx")
    params = dict(m.named_parameters())
    for k in keys:
        _close(params[k].grad.numpy(), GOLD[pre + "grad__" + k], 2e-5, k)


# ---- sequence encoders inside DEEP groups (dbmtl_taobao_seq) ---------------------------------------------------------
@pytest.mark.parametrize("jagged", ["1", "0"])
def test_seq_example_builds_and_trains(jagged, monkeypatch):
    """dbmtl_taobao_seq.config as stored: group `all` = 16 features (256) + the DIN encoder over click_50_seq (48);
    the encoder reads jagged rows by default, the padded form with TZK_DIN_JAGGED=0; two CPU steps lower the loss."""
    from oracle_backend import OracleKernels

    monkeypatch.setenv("TZK_DIN_JAGGED", jagged)
    pipe = Pipeline(os.path.join(REF_EXAMPLES, "dbmtl_taobao_seq.config"), device="cpu", max_rows=200, seed=3)
    eg = pipe.model.embedding_group
    assert eg.group_total_dim("all") == 16 * 16 + 48
    assert eg.group_feature_dims("all")["all_seq_encoder_0"] == 48
    enc = eg._group_name_to_seq_encoders["all"][0]
    assert enc.mlp.hidden_units == [32, 8] and enc.mlp.mlp[0].perceptron[0].weight.shape == (32, 4 * 48)
    jag = any(getattr(impl, "_jagged_for_attention", None) for impl in eg.seq_emb_impls.values())
    assert jag == (jagged == "1")
    batch = pipe.synthetic_batch(24, seed=1)
    with Fn.use_backend(OracleKernels()):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all() and l1 < l0


def test_other_deep_group_encoders_raise():
    text = GENERATORS["dbmtl_taobao_seq"]()
    with pytest.raises(NotImplementedError, match="simple_attention"):
        _model(text.replace("din_encoder {", "simple_attention {").replace(
            "                attn_mlp {\n                    hidden_units: [32, 8]\n                }\n", ""))


# ---- session ids are grouped by their full value ---------------------------------------------------------------------
def test_session_ids_beyond_the_table_and_negative(kern):
    """Raw session ids need not lie in the feature's table: the grouping uses every bit (the model passes 64 key bits),
    so ids that share their low bits stay apart and negative ids group."""
    logits, y, _, _ = R.seeded_case("mixed")
    B = len(y)
    rng = np.random.default_rng(3)
    base = rng.integers(0, 6, B)
    s = np.where(base % 2 == 0, base + (1 << 40), -base - 7).astype(np.int64)   # same low bits, different ids
    want_loss, want_d = R.jrc(logits, y, s, 0.5)
    loss, d = _run_kernel(kern, logits, y, s, None, 0.5)
    _close(loss, want_loss, 1e-5)
    np.testing.assert_allclose(d, want_d, rtol=0, atol=1e-5 * np.abs(want_d).max())
    _close(Fn.jrc_loss(torch.tensor(logits), torch.tensor(y), torch.tensor(s), 0.5).item(), want_loss, 1e-6)


def test_synthetic_sessions_bounded_by_the_table():
    from torcheasyrec_b200.features import BASE_DATA_GROUP

    pipe = Pipeline(os.path.join(REF_EXAMPLES, "dbmtl_taobao_jrc.config"), device="cpu", max_rows=5, seed=3)
    sid = pipe.synthetic_batch(256, seed=1).sparse_features[BASE_DATA_GROUP].to_dict()["user_id"].values()
    assert int(sid.max()) < 5


def test_pareto_refused_by_dbmtl_only():
    text = "model_config {\n    use_pareto_loss_weight: true\n"
    with pytest.raises(NotImplementedError, match="pareto"):
        _model(GENERATORS["dbmtl_taobao"]().replace("model_config {\n", text))
    _model(GENERATORS["mmoe_taobao"]().replace("model_config {\n", text))     # ignored there, as before


# ---- data parallelism over gloo --------------------------------------------------------------------------------------
def test_dbmtl_taobao_two_ranks_equal_the_unsharded_twin():
    from test_distributed_cpu import _run

    _run(2, os.path.join(REF_EXAMPLES, "dbmtl_taobao.config"), "mixed", rw_min_rows=250)


def _jrc_worker(rank, world, port, path, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    try:
        from torcheasyrec_b200.distributed import DenseGradSync, shard_model
        from torcheasyrec_b200.rank_models import dense_optimizer_from_config

        with Fn.use_backend(JrcOracleKernels()):
            ref = Pipeline(path, device="cpu", max_rows=300, seed=5, capturable=False)
            shd = Pipeline(path, device="cpu", max_rows=300, seed=5, capturable=False)
            shd.model.load_state_dict(ref.model.state_dict())
            shard_model(shd.model, torch.device("cpu"), default="mixed", rw_min_rows=250, source=ref.model)
            shd.model.set_sparse_optimizer(ref.model.sparse_collections()[0].optimizer)
            shd.dense_optimizer = dense_optimizer_from_config(shd.cfg.train_config, shd.model.dense_parameters())
            shd.grad_sync = DenseGradSync(shd.model.dense_parameters())
            batches = [ref.synthetic_batch(48, seed=77 + r) for r in range(world)]
            # the unsharded twin on each rank's half: per-half losses, and the mean of the halves' dense gradients
            ref.dense_optimizer.zero_grad(set_to_none=True)
            halves = [ref.train_wrapper(b)[0] for b in batches]
            (sum(halves) / world).backward()
            want = {n: p.grad.detach().clone() for n, p in ref.model.named_parameters()
                    if p.grad is not None and not n.startswith("embedding_group")}
            loss = shd.eager_step(batches[rank])
        np.testing.assert_allclose(float(loss), float(halves[rank]), rtol=1e-6)
        got = {n: p.grad for n, p in shd.model.named_parameters() if n in want}
        assert set(got) == set(want) and want
        for n in want:
            np.testing.assert_allclose(got[n].numpy(), want[n].numpy(), rtol=1e-5, atol=1e-7, err_msg=n)
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_jrc_two_ranks_each_loss_over_its_own_half():
    """dbmtl_taobao_jrc over gloo W = 2: each rank's loss is JRC over its own half (sessions never span ranks, as in
    the reference), and the synced dense gradients are the mean of the two halves' gradients."""
    import torch.multiprocessing as mp
    from test_distributed_cpu import _free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    path = os.path.join(REF_EXAMPLES, "dbmtl_taobao_jrc.config")
    procs = [ctx.Process(target=_jrc_worker, args=(r, 2, port, path, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    bad = [r for r in res if r[1] != "ok"]
    assert not bad, "\n".join(f"rank {r}: {m}" for r, m in bad)
