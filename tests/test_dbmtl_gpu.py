"""The JRC loss kernel (csrc/tzk_jrc.cuh) on the H100: against the float64 restatement over batch sizes and session
lengths, bit-identical reruns and graph replays, the fused model path against the torch formulation, and the JRC
example trained as captured steps."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402

pytestmark = pytest.mark.gpu
REF_EXAMPLES = os.path.join(HERE, "golden", "ref_examples")


def _f64(logits, y, s, alpha, w=None):
    """Float64 O(B) restatement on the GPU (functional.torch_jrc_loss), for sizes where [B, B] masks do not fit."""
    lg = logits.double().requires_grad_(True)
    loss = Fn.torch_jrc_loss(lg, y.double(), s, alpha, "mean" if w is None else "none")
    if w is not None:
        loss = (loss * w.double()).mean()
    loss.backward()
    return loss.detach(), lg.grad


def _case(B, mean_len, seed, weighted=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(B, 2, device="cuda", generator=g) * 2
    y = (torch.rand(B, device="cuda", generator=g) < 0.3).float()
    n_sess = max(1, B // mean_len)
    s = torch.randint(0, n_sess, (B,), device="cuda", generator=g) * 7919 + 3
    w = torch.rand(B, device="cuda", generator=g) * 2 if weighted else None
    return logits, y, s, w


@pytest.mark.parametrize("B", [1, 7, 8192, 65536, 200000])   # 200000: carry over 4 tiles of chunks
@pytest.mark.parametrize("mean_len", [1, 8, 64, "B"])
def test_kernel_matches_float64(B, mean_len):
    L = B if mean_len == "B" else mean_len
    for weighted in (False, True):
        logits, y, s, w = _case(B, L, seed=B + (L if isinstance(L, int) else 0), weighted=weighted)
        loss, d = default_kernels().jrc_loss(logits, y, s, w, 0.5)
        want_loss, want_d = _f64(logits, y, s, 0.5, w)
        if torch.isnan(want_loss):
            assert torch.isnan(loss)
        else:
            assert abs(loss.item() - want_loss.item()) <= 1e-5 * abs(want_loss.item()) + 1e-7
        assert torch.isfinite(d).all()
        err = (d.double() - want_d).abs().max().item()
        # one session of 200000: every pair combine rounds its shift (x.m - M) once, and the reduction is ~20 combines
        # deep (8 in the chunk, 8 per carry tile, one per tile); 1e-5 holds up to B = 65536 (DESIGN §5)
        tol = 5e-5 if B > 65536 and mean_len == "B" else 1e-5
        assert err <= tol * max(want_d.abs().max().item(), 1e-30), err


def test_kernel_bits_repeat_and_graph_replay():
    logits, y, s, _ = _case(65536, 8, seed=1)
    K = default_kernels()
    l1, d1 = K.jrc_loss(logits, y, s, None, 0.3, 27)
    l2, d2 = K.jrc_loss(logits, y, s, None, 0.3, 27)
    assert torch.equal(l1, l2) and torch.equal(d1, d2)
    K.jrc_loss(logits, y, s, None, 0.3, 27)       # workspace allocated before capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lg, dg = K.jrc_loss(logits, y, s, None, 0.3, 27)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(lg, l1) and torch.equal(dg, d1)


def test_fused_path_matches_torch_path():
    logits, y, s, _ = _case(8192, 8, seed=3)
    a = logits.clone().requires_grad_(True)
    la = Fn.jrc_loss(a, y, s, 0.5)
    la.backward()
    b = logits.clone().requires_grad_(True)
    lb = Fn.torch_jrc_loss(b, y, s, 0.5)
    lb.backward()
    torch.testing.assert_close(la, lb, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(a.grad, b.grad, rtol=1e-4, atol=1e-5 * b.grad.abs().max().item())


def test_single_class_nan_and_bad_label_on_device():
    logits, y, s, _ = _case(1000, 8, seed=4)
    loss, d = default_kernels().jrc_loss(logits, torch.zeros_like(y), s, None, 0.5)
    assert torch.isnan(loss) and torch.isfinite(d).all()
    y2 = y.clone()
    y2[10] = 2.0
    loss, d = default_kernels().jrc_loss(logits, y2, s, None, 0.5)
    assert torch.isnan(loss) and torch.isnan(d[10]).all()
    loss, _ = default_kernels().jrc_loss(logits[:0], y[:0], s[:0], None, 0.5)
    assert torch.isnan(loss)


def test_jrc_example_trains_captured():
    """dbmtl_taobao_jrc.config as stored, as a captured step on a repeated batch: finite losses that go down."""
    from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

    p = Pipeline(os.path.join(REF_EXAMPLES, "dbmtl_taobao_jrc.config"), device="cuda", max_rows=2000, seed=21)
    batch = p.synthetic_batch(8192, seed=2)
    step = GraphedTrainStep(p, batch, warmup=2)
    losses = []
    for _ in range(6):
        step.load(batch.pin_memory())
        losses.append(float(step.replay()))
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_seq_example_trains():
    """dbmtl_taobao_seq.config as stored (DIN encoder inside group `all`, jagged rows) on the GPU: finite losses that go
    down on a repeated batch.  Eager steps, as for every sequence workload here (engine.py): the query of a multi-value
    id feature is pooled with ATen's segment_reduce, which a CUDA graph cannot capture."""
    from torcheasyrec_b200.engine import Pipeline

    p = Pipeline(os.path.join(REF_EXAMPLES, "dbmtl_taobao_seq.config"), device="cuda", max_rows=2000, seed=21)
    batch = p.synthetic_batch(2048, seed=2).to("cuda")
    losses = [float(p.eager_step(batch)) for _ in range(6)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_session_ids_use_all_64_bits():
    """Ids that share their low bits, ids past any table and negative ids form the sessions their full values say."""
    logits, y, s, _ = _case(8192, 8, seed=6)
    s = torch.where(s % 2 == 0, s + (1 << 40), -s - 7)
    loss, d = default_kernels().jrc_loss(logits, y, s, None, 0.5)
    want_loss, want_d = _f64(logits, y, s, 0.5)
    assert abs(loss.item() - want_loss.item()) <= 1e-5 * abs(want_loss.item())
    assert (d.double() - want_d).abs().max().item() <= 1e-5 * want_d.abs().max().item()
