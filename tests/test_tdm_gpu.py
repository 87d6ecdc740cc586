"""TDM on the H100: both fused multi-window DIN kernels against float64 over shapes in their cover, bit-identical
reruns, the fused encoder against the torch jagged formulation, the stored example trained and evaluated, and the
torch path under BF16 autocast and outside the cover."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import tdm_ref as R  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402
from torcheasyrec_b200.rank_models import MultiWindowDINEncoder  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF_EXAMPLE = os.path.join(HERE, "golden", "ref_examples", "tdm_taobao.config")
EXAMPLE_WINDOWS = [1, 1, 1, 2, 2, 2, 5, 6, 10, 20]


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, np.abs(want).max() if want.size else 1.0), err_msg=name)


def _run(case, windows, dout):
    q, seq, off, layers, lw, lb, aw = case
    prelu = layers[0][2] is not None
    c = lambda t: None if t is None else t.float().to(DEV).contiguous()  # noqa: E731
    lay = [tuple(c(t) for t in l) for l in layers]
    offs = torch.from_numpy(off).to(DEV)
    k = default_kernels()
    out, z = k.tdm_fwd(c(q), c(seq), offs, lay, c(lw).reshape(1, -1), c(lb), c(aw), windows, prelu)
    d_q, d_seq, grads, d_lw, d_lb, d_aw = k.tdm_bwd(c(q), c(seq), offs, lay, c(lw).reshape(1, -1), c(lb), c(aw),
                                                    windows, prelu, z, c(dout))
    flat = []
    for dw, db, ds in grads:
        flat += [dw, db] + ([ds] if prelu else [])
    torch.cuda.synchronize()
    return out, z, d_q, d_seq, flat + [d_lw.reshape(-1), d_lb, d_aw]


def _reference(case, windows, seed=0):
    q, seq, off, layers, lw, lb, aw = case
    lens_np = off[1:] - off[:-1]
    seqp, lens = R.pad_rows(seq, off, T=max(int(lens_np.max()) if len(lens_np) else 0, 1))
    kind = "relu" if layers[0][2] is None else "prelu"
    leaves = [q, seqp, lw, lb, aw] + [t for l in layers for t in l if t is not None]
    for t in leaves:
        t.requires_grad_(True)
    out = R.multiwindow_din(q, seqp, lens, windows, layers, kind, lw, lb, aw)
    dout = torch.from_numpy(np.random.default_rng(seed).standard_normal(tuple(out.shape)))
    out.backward(dout)
    rows = torch.cat([seqp.grad[b, :int(n)] for b, n in enumerate(lens_np)] +
                     [torch.zeros(0, seq.shape[1], dtype=torch.float64)])
    grads = []
    for W, b, s in layers:
        grads += [W.grad, b.grad] + ([s.grad] if s is not None else [])
    return out.detach(), dout, q.grad, rows, grads + [lw.grad, lb.grad, aw.grad]


SHAPES = {
    "example": (48, 48, [36], "prelu", EXAMPLE_WINDOWS, 3000, 60),
    "relu_84": (16, 16, [8, 4], "relu", [1, 2, 5], 1000, 12),
    "three_layers_dq": (64, 40, [32, 16, 8], "prelu", [4, 4, 8, 16], 700, 40),
    "widest": (128, 128, [40], "relu", [64, 64, 128], 300, 270),
    "units64": (64, 64, [64, 64], "relu", [1, 2, 5], 400, 12),
    "all_zero_lengths": (8, 8, [4], "prelu", [1, 1], 50, 0),
}


@pytest.mark.parametrize("tag", list(SHAPES))
def test_kernels_against_float64(tag):
    C, Dq, hidden, kind, windows, B, mx = SHAPES[tag]
    case = R.case(len(tag), B, C, Dq, hidden, windows, kind, mx, [0] * B if mx == 0 else None)
    out_r, dout, dq_r, dseq_r, grads_r = _reference(case, windows)
    out, _, dq, dseq, grads = _run(case, windows, dout)
    _close(out.cpu().double(), out_r, 1e-5, "out")
    _close(dq.cpu().double(), dq_r, 1e-5, "d_query")
    _close(dseq.cpu().double(), dseq_r, 1e-5, "d_seq")
    for i, (g, r) in enumerate(zip(grads, grads_r)):
        _close(g.cpu().double().reshape(-1), r.reshape(-1), 5e-5, f"dparam{i}")


def test_reruns_bit_identical():
    windows = EXAMPLE_WINDOWS
    case = R.case(3, 5000, 48, 48, [36], windows, "prelu", 50)
    dout = torch.randn(5000, 11 * 48, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    a, b = _run(case, windows, dout), _run(case, windows, dout)
    for x, y in zip(torch.utils._pytree.tree_leaves(a), torch.utils._pytree.tree_leaves(b)):
        assert torch.equal(x, y)


def _encoder_inputs(B, C, Dq, mx, seed):
    g = torch.Generator().manual_seed(seed)
    kind = torch.randint(0, 4, (B,), generator=g)
    lens = torch.where(kind == 0, 0, torch.where(kind == 1, 1, torch.where(kind == 2, torch.randint(2, mx + 1, (B,),
                                                                                                   generator=g), mx)))
    off = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lens, 0)])
    q = torch.randn(B, Dq, generator=g) * 0.5
    seq = torch.randn(int(off[-1]), C, generator=g) * 0.5
    return q.to(DEV), seq.to(DEV), off.to(DEV), lens.to(DEV)


def test_fused_encoder_against_torch_jagged():
    torch.manual_seed(0)
    enc = MultiWindowDINEncoder(48, 48, "seq", EXAMPLE_WINDOWS, dict(hidden_units=[36], activation="nn.PReLU")).to(DEV)
    q, seq, off, lens = _encoder_inputs(4096, 48, 48, 50, 1)
    emb = {"seq.query": q, "seq.sequence": seq, "seq.sequence_length": lens, "seq.sequence_offsets": off}
    assert Fn.multiwindow_din_usable(q, seq, enc.mlp, EXAMPLE_WINDOWS)
    outs = []
    for fused in (True, False):
        qq, ss = q.clone().requires_grad_(True), seq.clone().requires_grad_(True)
        enc.zero_grad(set_to_none=True)
        e = dict(emb, **{"seq.query": qq, "seq.sequence": ss})
        y = enc(e) if fused else Fn.torch_multiwindow_din(qq, ss, off, enc.mlp, enc.linear, enc.active, EXAMPLE_WINDOWS)
        y.backward(torch.ones_like(y))
        outs.append([y.detach(), qq.grad, ss.grad] + [p.grad.clone() for p in enc.parameters()])
    for i, (a, b) in enumerate(zip(*outs)):
        _close(a.cpu(), b.cpu(), 1e-4, f"tensor{i}")


def test_example_trains_and_evaluates_on_the_gpu():
    pipe = Pipeline(REF_EXAMPLE, device="cuda:0", max_rows=100000, seed=3, capturable=False)
    assert type(pipe.model).__name__ == "TDM"
    k = default_kernels()
    batch = pipe.synthetic_batch(2048, seed=1).to("cuda:0")
    n0 = k.launches
    ls = [float(pipe.eager_step(batch)) for _ in range(4)]
    assert k.launches > n0
    assert np.isfinite(ls).all() and ls[-1] < ls[0]
    m = pipe.evaluate([pipe.synthetic_batch(1024, seed=s).to("cuda:0") for s in range(3)])
    assert set(m) == {"auc", "softmax_cross_entropy"}
    assert 0.0 <= m["auc"] <= 1.0 and np.isfinite(m["softmax_cross_entropy"])


def test_bf16_autocast_and_outside_cover_take_the_torch_path(monkeypatch):
    calls = []
    monkeypatch.setattr(Fn, "torch_multiwindow_din",
                        (lambda f: (lambda *a, **k: calls.append(1) or f(*a, **k)))(Fn.torch_multiwindow_din))
    torch.manual_seed(0)
    enc = MultiWindowDINEncoder(48, 48, "seq", EXAMPLE_WINDOWS, dict(hidden_units=[36], activation="nn.PReLU")).to(DEV)
    q, seq, off, lens = _encoder_inputs(256, 48, 48, 50, 2)
    emb = {"seq.query": q, "seq.sequence": seq, "seq.sequence_length": lens, "seq.sequence_offsets": off}
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = enc(emb)
    assert calls == [1] and y.dtype == torch.float32 and torch.isfinite(y).all()
    wide = MultiWindowDINEncoder(48, 48, "seq", EXAMPLE_WINDOWS, dict(hidden_units=[80])).to(DEV)   # > 64 units
    assert not Fn.multiwindow_din_usable(q, seq, wide.mlp, EXAMPLE_WINDOWS)
    wide(emb)
    odd = MultiWindowDINEncoder(48, 48, "seq", [100, 200], dict(hidden_units=[8])).to(DEV)       # S > 256
    odd(emb)
    assert calls == [1, 1, 1]
