"""Sequence encoders on the H100: the fused self-attention and pooling kernels (csrc/tzk_seq_attn.cuh) against float64
over shapes in their cover and at B = 8192 with the default 512 / 8, the encoders on the fused and torch paths, a
captured forward + backward replayed to the eager bits, bit-identical reruns, and dbmtl_taobao_seq_encoders trained on
the fused path."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import seq_encoder_ref as R  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.kernels import default_kernels  # noqa: E402
from torcheasyrec_b200.rank_models import PoolingEncoder, SelfAttentionEncoder  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, np.abs(want).max() if want.size else 1.0), err_msg=name)


def _np(t):
    return t.detach().double().cpu().numpy()


def _lengths(B, seed, cap=100):
    """SURVEY's cfg4 mixture: 0, 1, U[2, cap] and cap, a quarter each."""
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 4, B)
    return np.where(kind == 0, 0, np.where(kind == 1, 1, np.where(kind == 2, rng.integers(2, cap + 1, B), cap)))


def _case(lengths, E, seed):
    g = torch.Generator().manual_seed(seed)
    N = int(np.sum(lengths))
    q, k, v = (torch.randn(N, E, generator=g, dtype=torch.float64).to(DEV) for _ in range(3))
    dout = torch.randn(len(lengths), E, generator=g, dtype=torch.float64).to(DEV)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)).to(DEV)
    return q, k, v, off, dout


def _fused(q, k, v, off, H, mx, dout):
    kk = default_kernels()
    f = [t.float().contiguous() for t in (q, k, v)]
    pooled, lse = kk.self_attn_pool_fwd(*f, off, H, mx)
    return pooled, kk.self_attn_pool_bwd(*f, off, H, mx, lse, dout.float().contiguous())


def _float64(q, k, v, off, H, mx, dout, batched):
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    fn = Fn.torch_self_attn_pool if batched else R.self_attn_pool
    out = fn(*leaves, off, H, mx)
    out.backward(dout)
    return out.detach(), [t.grad for t in leaves]


# (lengths, E, H, max_len)
SHAPES = {
    "ref_test": ([0, 1, 70, 5, 33], 32, 4, 0),
    "default": ([3, 0, 1, 66, 20, 9, 100, 130], 512, 8, 0),
    "one_head": ([4, 9, 0, 1], 16, 1, 0),
    "hd_1": ([5, 0, 3, 1], 4, 4, 0),
    "hd_128": ([70, 9, 0, 200], 256, 2, 0),
    "crop": ([7, 3, 0, 5, 2, 9, 80], 16, 2, 3),
    "crop_across_tiles": ([150, 70, 0], 64, 4, 66),
}


@pytest.mark.parametrize("tag", list(SHAPES))
def test_attention_kernels_against_float64(tag):
    lengths, E, H, mx = SHAPES[tag]
    q, k, v, off, dout = _case(lengths, E, len(tag))
    out_r, grads_r = _float64(q, k, v, off, H, mx, dout, batched=False)
    pooled, grads = _fused(q, k, v, off, H, mx, dout)
    _close(_np(pooled), _np(out_r), 1e-5, "pooled")
    for g, r, nm in zip(grads, grads_r, ("dq", "dk", "dv")):
        _close(_np(g), _np(r), 2e-5, nm)


@pytest.mark.parametrize("E,H", [(512, 8), (64, 4)])
def test_attention_kernels_at_batch_8192(E, H):
    """B = 8192 over the cfg4 length mixture against the float64 torch formulation (validated against the per-sample
    restatement on the CPU)."""
    q, k, v, off, dout = _case(_lengths(8192, 1), E, 2)
    out_r, grads_r = _float64(q, k, v, off, H, 0, dout, batched=True)
    pooled, grads = _fused(q, k, v, off, H, 0, dout)
    _close(_np(pooled), _np(out_r), 1e-5, "pooled")
    for g, r, nm in zip(grads, grads_r, ("dq", "dk", "dv")):
        _close(_np(g), _np(r), 2e-5, nm)


def test_attention_reruns_and_graph_replay_bit_identical():
    q, k, v, off, dout = _case(_lengths(512, 3), 64, 4)
    f = [t.float().contiguous() for t in (q, k, v)]
    d = dout.float().contiguous()
    kk = default_kernels()

    def step():
        pooled, lse = kk.self_attn_pool_fwd(*f, off, 4, 0)
        return (pooled,) + tuple(kk.self_attn_pool_bwd(*f, off, 4, 0, lse, d))

    a, b = step(), step()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, captured))


@pytest.mark.parametrize("mean,mx", [(True, 0), (False, 0), (True, 30), (False, 30)])
def test_pool_kernels_against_float64(mean, mx):
    lengths = _lengths(8192, 5)
    g = torch.Generator().manual_seed(6)
    seq = torch.randn(int(lengths.sum()), 48, generator=g, dtype=torch.float64).to(DEV)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)).to(DEV)
    dout = torch.randn(len(lengths), 48, generator=g, dtype=torch.float64).to(DEV)
    leaf = seq.clone().requires_grad_(True)
    want = Fn.torch_jagged_pool(leaf, off, mx, mean)
    want.backward(dout)
    kk = default_kernels()
    _close(_np(kk.jagged_pool_fwd(seq.float(), off, mx, mean)), _np(want), 1e-6, "out")
    _close(_np(kk.jagged_pool_bwd(dout.float(), off, seq.shape[0], mx, mean)), _np(leaf.grad), 1e-6, "d_seq")


@pytest.mark.parametrize("E,H,mx", [(512, 8, 0), (64, 4, 20)])
def test_encoders_fused_and_torch_paths_agree(E, H, mx, monkeypatch):
    lengths = _lengths(1024, 7)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)).to(DEV)
    seq0 = torch.randn(int(lengths.sum()), 48, generator=torch.Generator().manual_seed(8)).to(DEV)
    emb = {"s.sequence_length": torch.from_numpy(lengths).to(DEV), "s.sequence_offsets": off}
    torch.manual_seed(0)
    enc = SelfAttentionEncoder(48, "s", E, num_heads=H, max_seq_length=mx).to(DEV)
    res = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setattr(Fn, "self_attn_pool_usable", lambda *a: False)
        enc.zero_grad()
        seq = seq0.clone().requires_grad_(True)
        out = enc(dict(emb, **{"s.sequence": seq}))
        out.square().sum().backward()
        res.append([out.detach(), seq.grad] + [p.grad.clone() for p in enc.parameters()])
    for i, (a, b) in enumerate(zip(*res)):
        assert torch.isfinite(a).all()
        _close(_np(a), _np(b), 1e-4, f"tensor {i}")
    pool = PoolingEncoder(48, "s", pooling_type="mean", max_seq_length=mx)
    s1 = seq0.clone().requires_grad_(True)
    torch.testing.assert_close(pool(dict(emb, **{"s.sequence": s1})),
                               Fn.torch_jagged_pool(seq0, off, mx, True), rtol=1e-6, atol=1e-6)


def test_seq_encoders_config_trains_on_the_fused_path(monkeypatch):
    calls = {"attn": 0, "pool": 0}
    attn, pool = Fn.self_attn_pool, Fn.jagged_pool

    def count_attn(*a, **k):
        calls["attn"] += 1
        return attn(*a, **k)

    def count_pool(*a, **k):
        calls["pool"] += 1
        return pool(*a, **k)

    monkeypatch.setattr(Fn, "self_attn_pool", count_attn)
    monkeypatch.setattr(Fn, "jagged_pool", count_pool)
    pipe = Pipeline("dbmtl_taobao_seq_encoders", device="cuda:0", max_rows=100000, seed=3, capturable=False)
    batch = pipe.synthetic_batch(2048, seed=1).to("cuda:0")
    ls = [float(pipe.eager_step(batch)) for _ in range(3)]
    assert np.isfinite(ls).all() and ls[-1] < ls[0]
    assert calls == {"attn": 3, "pool": 3}
