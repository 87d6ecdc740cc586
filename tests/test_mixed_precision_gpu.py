"""train_config.mixed_precision on the H100: the BF16 DLRM-Criteo interaction kernels against the float64 restatement of
tests/test_mixed_precision_cpu.py (same rounding-point bounds, derived there), the kernel path against the pure-torch
autocast path (TZK_INTERACT_BF16=0, the reference's formulation), CUDA-graph replay against the eager step, and BF16 /
FP16 steps of the other example models.

Tolerance of the kernel path against the torch path (both bf16 autocast): X agrees within the pair bound (one bf16 ulp
plus the fp32 accumulation term) because both accumulate exact bf16 products in fp32 and round once.  Downstream, each
bf16 GEMM output (three final-MLP layers, the backward's dX and dW) may round one ulp differently where its fp32 input
differs, so values derived from X carry at most a few bf16 ulps of their magnitude: logits and loss are held to TOL = 2^-5 (4 bf16
ulps) of each tensor's largest magnitude.  Gradients are held to TOL in norm (||a - b|| <= TOL ||b||): a ReLU gate whose
pre-activation lies within an ulp of zero may open on one path only and change that sample's gradient outright.  After two training steps the
tables are held to TOL of their largest magnitude.  The dense parameters' changes are held in norm to 4 TOL: Adam divides
each element's step by that element's own gradient RMS, which magnifies the relative difference of small gradient
elements; no element may move by more than the 4 lr two Adam steps allow."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_mixed_precision_cpu import ROW, bf16_bits, bits_f, check_bwd, check_fwd  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 2.0 ** -5


def _kernels():
    from torcheasyrec_b200.kernels import default_kernels

    return default_kernels()


def _bf16_tensor(bits):
    return torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16)


def _bits(t):
    return t.detach().cpu().view(torch.int16).numpy().view(np.uint16)


@pytest.mark.parametrize("B", [300, 65541])
def test_bf16_kernels_match_float64_restatement(B):
    rng = np.random.default_rng(B)
    dense_bits = bf16_bits(rng.standard_normal((B, 16)))
    sparse = rng.standard_normal((B, 416)).astype(np.float32)
    d_out_bits = bf16_bits(rng.standard_normal((B, ROW)))
    d_out_bits[:, 351] = 0
    dense = _bf16_tensor(dense_bits).cuda()
    sp = torch.from_numpy(sparse).cuda()
    x = _kernels().dot_interact27_fwd_bf16(dense, sp)
    check_fwd(_bits(x), dense_bits, sparse)
    dd, ds = _kernels().dot_interact27_bwd_bf16(_bf16_tensor(d_out_bits).cuda(), dense, sp)
    check_bwd(_bits(dd), ds.cpu().numpy(), d_out_bits, dense_bits, sparse)


def test_bf16_kernels_reject_what_they_do_not_cover():
    from torcheasyrec_b200 import _lib
    from torcheasyrec_b200.kernels import TzkError, _stream

    k = _kernels()
    B = 64
    dense = torch.zeros((B, 16), dtype=torch.bfloat16, device="cuda")
    sparse = torch.zeros((B, 416), device="cuda")
    with pytest.raises(TzkError):                                  # short rows
        k.dot_interact27_fwd_bf16(dense, torch.zeros((B, 400), device="cuda"))
    with pytest.raises(TzkError):                                  # fp32 dense
        k.dot_interact27_fwd_bf16(dense.float(), sparse)
    buf = torch.zeros((B, 420), device="cuda")
    with pytest.raises(TzkError, match="16-B aligned"):            # sparse rows 4 B off alignment
        k.dot_interact27_fwd_bf16(dense, buf[:, 1:417])
    dbuf = torch.zeros((B, 18), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(TzkError, match="8-B aligned"):             # dense row stride not a multiple of 4
        k.dot_interact27_fwd_bf16(dbuf[:, :16], sparse)
    L = _lib.lib()
    out = torch.zeros((B, ROW), dtype=torch.bfloat16, device="cuda")
    assert L.tzk_dot_interact27_fwd_bf16(dense.data_ptr(), 16, sparse.data_ptr(), 416, B, out.data_ptr(), 780,
                                         _stream()) != 0      # output row shorter than 784
    assert L.tzk_dot_interact27_fwd_bf16(dense.data_ptr(), 16, sparse.data_ptr(), 416, -1, out.data_ptr(), ROW,
                                         _stream()) != 0      # negative batch
    with pytest.raises(TzkError):                                  # dX of the wrong width
        k.dot_interact27_bwd_bf16(out[:, :700], dense, sparse)
    torch.cuda.synchronize()


def _bf16_pipe(seed=3, **kw):
    from torcheasyrec_b200.engine import Pipeline

    return Pipeline("dlrm_criteo", device="cuda:0", max_rows=5000, seed=seed,
                    edits={"train_config.mixed_precision": "BF16"}, **kw)


def _close(a, b, what):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    lim = TOL * float(b.abs().max()) + 1e-30
    assert float((a - b).abs().max()) <= lim, (what, float((a - b).abs().max()), lim)


def _close_norm(a, b, what):
    """||a - b|| <= TOL ||b||: for gradients, where a ReLU gate whose pre-activation lies within a bf16 ulp of zero may
    open on one path and not the other, which changes that sample's gradient through the gate entirely."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert float((a - b).norm()) <= TOL * float(b.norm()), (what, float((a - b).norm()), float(b.norm()))


def test_interaction_x_kernel_vs_torch_autocast():
    """X of the kernel and of the torch autocast path (cuBLAS bf16 bmm) on the same inputs: copied columns bit-equal, each
    pair within the forward bound of both against bf16(exact), so within twice that of each other."""
    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.dense_gemm import InteractBf16Fn
    from test_mixed_precision_cpu import fwd_reference, ulp

    rng = np.random.default_rng(0)
    B = 4096
    dense_bits = bf16_bits(rng.standard_normal((B, 16)))
    sparse_np = rng.standard_normal((B, 416)).astype(np.float32)
    dense, sparse = _bf16_tensor(dense_bits).cuda(), torch.from_numpy(sparse_np).cuda()
    with torch.autocast("cuda", torch.bfloat16):
        xk = InteractBf16Fn.apply(dense, sparse)
        xt, in_map = Fn.dlrm_interaction(dense, sparse, 26, 16, aligned=True)
    assert in_map is None and xk.dtype == torch.bfloat16 and xt.dtype == torch.float32 and xt.shape == (B, 783)
    xk = xk.float()
    xk = torch.cat([xk[:, :351], xk[:, 352:]], dim=1).cpu().double().numpy()
    xt = xt.cpu().double().numpy()
    np.testing.assert_array_equal(xk[:, 351:367], xt[:, 351:367])                   # dense: bf16 on both paths
    # sparse: the kernel writes bf16(sparse); the torch path keeps fp32 there and the first Linear rounds it to bf16
    np.testing.assert_array_equal(xk[:, 367:], bits_f(bf16_bits(xt[:, 367:].astype(np.float32))))
    ref, A, _ = fwd_reference(dense_bits, sparse_np)
    bound = 2 * (ulp(np.maximum(np.abs(xk[:, :351]), np.abs(xt[:, :351]))) + 2.0 ** -19 * A)
    assert np.all(np.abs(xk[:, :351] - xt[:, :351]) <= bound)


def _twin_steps(env_value, steps=2, B=4096):
    os.environ["TZK_INTERACT_BF16"] = env_value
    try:
        p = _bf16_pipe(seed=7, capturable=False)
        batch = p.synthetic_batch(B, seed=11).to("cuda:0")
        p0 = {k: v.detach().clone() for k, v in p.model.named_parameters()}
        # first step by hand: logits, loss and gradients
        p.dense_optimizer.zero_grad(set_to_none=True)
        sparse_grads = {}
        build_input = p.model.build_input

        def hooked(bt):       # the pooled-embedding gradient d_sparse, as the fused sparse backward receives it
            g = build_input(bt)
            g[p.model._sparse_group_name].register_hook(lambda gr: sparse_grads.__setitem__("d", gr.detach().clone()))
            return g

        p.model.build_input = hooked
        total, (_, preds, _) = p.train_wrapper(batch)
        total.backward()
        p.model.build_input = build_input
        grads = {k: v.grad.detach().clone() for k, v in p.model.named_parameters() if v.grad is not None}
        p.dense_optimizer.step()
        for _ in range(steps - 1):
            p.eager_step(batch)
        tables = [c.weights.detach().clone() for c in p.model.sparse_collections()]
        dense_ids = {id(v) for v in p.model.dense_parameters()}
        params = {k: v.detach().clone() for k, v in p.model.named_parameters() if id(v) in dense_ids}
        return dict(logits=preds["logits"], loss=total.detach(), grads=grads, tables=tables, params=params, p0=p0,
                    lr=max(g["lr"] for g in p.dense_optimizer.param_groups), sparse_grads=sparse_grads)
    finally:
        os.environ.pop("TZK_INTERACT_BF16", None)


def test_dlrm_bf16_kernel_path_matches_torch_autocast_path():
    k, t = _twin_steps("1"), _twin_steps("0")
    _close(k["logits"], t["logits"], "logits")
    _close(k["loss"], t["loss"], "loss")
    _close_norm(k["sparse_grads"]["d"], t["sparse_grads"]["d"], "d_sparse")
    assert set(k["grads"]) == set(t["grads"])
    for name in k["grads"]:
        _close_norm(k["grads"][name], t["grads"][name], name)
    for a, b in zip(k["tables"], t["tables"]):
        _close(a, b, "table")
    for name in k["params"]:
        da, db = k["params"][name] - k["p0"][name], t["params"][name] - t["p0"][name]
        diff = (da - db).abs()
        assert float(diff.max()) <= 4 * k["lr"] + 1e-12, name                   # two Adam steps move at most 2 lr each
        assert float(diff.double().norm()) <= 4 * TOL * float(db.double().norm()), name


def test_bf16_graph_replay_equals_eager_step():
    a = _bf16_pipe()
    batches = [a.synthetic_batch(1024, seed=40 + i) for i in range(3)]
    from torcheasyrec_b200.engine import GraphedTrainStep

    step = GraphedTrainStep(a, batches[0], warmup=2)
    b = _bf16_pipe()
    b.model.load_state_dict(a.model.state_dict())
    for ca, cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
        if ca.layout.interleaved:
            cb.weights.data.copy_(ca.weights.data)
        else:
            cb.opt_state.copy_(ca.opt_state)
    b.dense_optimizer.load_state_dict(copy.deepcopy(a.dense_optimizer.state_dict()))
    for bt in batches[1:]:
        step.load(bt.pin_memory())
        la = float(step.replay())
        lb = float(b.eager_step(bt.to("cuda:0")))
        assert la == lb
    for ca, cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
        assert torch.equal(ca.weights.data.view(torch.int32), cb.weights.data.view(torch.int32))
    for pa, pb in zip(a.model.dense_parameters(), b.model.dense_parameters()):
        assert torch.equal(pa.data, pb.data)


@pytest.mark.parametrize("name,mp", [("dlrm_criteo", "FP16"), ("deepfm_criteo", "BF16"), ("mmoe_taobao", "BF16"),
                                     ("deepfm_criteo", "FP16"), ("mmoe_taobao", "FP16"),
                                     ("multi_tower_din_taobao", "BF16"), ("multi_tower_din_taobao", "FP16")])
def test_mixed_precision_steps_of_the_example_models(name, mp):
    """A graphed step (eager for the sequence model, which the project always steps eagerly) with finite losses that
    move."""
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    p = Pipeline(name, device="cuda:0", max_rows=2000, seed=5, edits={"train_config.mixed_precision": mp})
    batches = [p.synthetic_batch(512, seed=60 + i) for i in range(3)]
    if any(f.is_sequence for f in p.features):
        losses = [float(p.eager_step(bt.to("cuda:0"))) for bt in batches]
    else:
        step = GraphedTrainStep(p, batches[0], warmup=2)
        losses = []
        for bt in batches:
            step.load(bt.pin_memory())
            losses.append(float(step.replay()))
    assert np.isfinite(losses).all() and len(set(losses)) > 1, losses
