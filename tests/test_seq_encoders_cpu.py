"""Sequence encoders of DEEP feature groups on the CPU: the SOURCE of the fused self-attention and pooling kernels
(csrc/tzk_seq_attn.cuh) run on the host through tests/native/cuda_cpu_shim.h against the float64 jagged restatement
(tests/seq_encoder_ref.py); that restatement and this repo's encoders against the reference's own
(tests/golden/ref_seq_encoders.npz); the factory, the schemas and the dbmtl_taobao_seq_encoders config."""
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
import seq_encoder_ref as R  # noqa: E402
from metric_oracle_backend import MetricOracleKernels  # noqa: E402

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200._lib import TzkJaggedPoolArgs, TzkSeqAttnArgs  # noqa: E402
from torcheasyrec_b200.config import parse_text  # noqa: E402
from torcheasyrec_b200.engine import Pipeline  # noqa: E402
from torcheasyrec_b200.example_configs import BUILTINS, EDITED_GENERATORS  # noqa: E402
from torcheasyrec_b200.rank_models import PoolingEncoder, SelfAttentionEncoder, _create_seq_encoder  # noqa: E402

NATIVE = os.path.join(HERE, "native")
GOLD = np.load(os.path.join(HERE, "golden", "ref_seq_encoders.npz"))


# ---- the kernel source on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kern(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libseq_attn_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", NATIVE,
                    "-x", "c++", os.path.join(NATIVE, "seq_attn_standalone.cu"), "-shared", "-fPIC", "-o", out],
                   check=True)
    L = ctypes.CDLL(out)
    P, I32 = ctypes.c_void_p, ctypes.c_int
    L.seq_attn_check.argtypes = [P, I32]
    for fn in ("self_attn_pool_fwd", "self_attn_pool_bwd", "jagged_pool_fwd", "jagged_pool_bwd"):
        getattr(L, fn).argtypes = [P, I32]
    return L


class ShimSeq:
    """self_attn_pool_* and jagged_pool_* of kernels.CudaKernels on CPU tensors, computed by the host build of the
    kernel source.  Grids: a fixed one, or min(work, 3) as a small stand-in for the device's."""

    def __init__(self, L, grid=None):
        self.L, self.grid, self.attn_calls, self.pool_calls = L, grid, 0, 0

    @staticmethod
    def args(q, k, v, offsets, H, max_len):
        a = TzkSeqAttnArgs()
        a.N, E = q.shape
        a.B, a.H, a.hd, a.max_len = offsets.numel() - 1, H, E // H, max_len
        a.ldq = a.ldk = a.ldv = E
        a.offsets, a.q, a.k, a.v = offsets.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr()
        return a

    def _grid(self, work):
        return self.grid or max(1, min(work, 3))

    def self_attn_pool_fwd(self, q, k, v, offsets, H, max_len):
        self.attn_calls += 1
        q, k, v = (t.detach().float().contiguous() for t in (q, k, v))
        self._keep = (q, k, v)
        a = self.args(q, k, v, offsets, H, max_len)
        pooled, lse = torch.empty(a.B, a.H * a.hd), torch.empty(a.N, a.H)
        a.pooled, a.lse = pooled.data_ptr(), lse.data_ptr()
        assert self.L.self_attn_pool_fwd(ctypes.byref(a), self._grid(a.B * a.H)) == 0
        return pooled, lse

    def self_attn_pool_bwd(self, q, k, v, offsets, H, max_len, lse, d_pooled):
        self.attn_calls += 1
        q, k, v = (t.detach().float().contiguous() for t in (q, k, v))
        d_pooled = d_pooled.float().contiguous()
        a = self.args(q, k, v, offsets, H, max_len)
        dq, dk, dv = (torch.empty_like(q) for _ in range(3))
        dsum = torch.empty(max(a.N * a.H, 1))
        a.lse, a.d_pooled, a.dsum = lse.data_ptr(), d_pooled.data_ptr(), dsum.data_ptr()
        a.dq, a.dk, a.dv = dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
        assert self.L.self_attn_pool_bwd(ctypes.byref(a), self._grid(a.B * a.H)) == 0
        return dq, dk, dv

    @staticmethod
    def pool_args(offsets, D, max_len, mean):
        a = TzkJaggedPoolArgs()
        a.B, a.D, a.max_len, a.mean = offsets.numel() - 1, D, max_len, int(mean)
        a.offsets = offsets.data_ptr()
        return a

    def jagged_pool_fwd(self, seq, offsets, max_len, mean):
        self.pool_calls += 1
        seq = seq.detach().float().contiguous()
        a = self.pool_args(offsets, seq.shape[1], max_len, mean)
        a.N = seq.shape[0]
        out = torch.empty(a.B, a.D)
        a.seq, a.out = seq.data_ptr(), out.data_ptr()
        assert self.L.jagged_pool_fwd(ctypes.byref(a), self._grid(-(-a.B // 8))) == 0
        return out

    def jagged_pool_bwd(self, d_out, offsets, N, max_len, mean):
        self.pool_calls += 1
        d_out = d_out.float().contiguous()
        a = self.pool_args(offsets, d_out.shape[1], max_len, mean)
        a.N = N
        d_seq = torch.empty(N, a.D)
        a.d_out, a.d_seq = d_out.data_ptr(), d_seq.data_ptr()
        assert self.L.jagged_pool_bwd(ctypes.byref(a), self._grid(-(-a.B // 8))) == 0
        return d_seq


class ShimBackend(MetricOracleKernels):
    """The CPU checker backend with the sequence encoders computed by the host build of their kernel source."""

    def __init__(self, L, grid=None):
        super().__init__()
        self.seq = ShimSeq(L, grid)
        for fn in ("self_attn_pool_fwd", "self_attn_pool_bwd", "jagged_pool_fwd", "jagged_pool_bwd"):
            setattr(self, fn, getattr(self.seq, fn))


def _close(got, want, r, name):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(np.asarray(got, np.float64), want, rtol=r,
                               atol=r * max(1.0, np.abs(want).max() if want.size else 1.0), err_msg=name)


def _np(t):
    return t.detach().double().numpy()


def _offsets(lengths):
    return torch.tensor(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64))


def _attn_case(seed, lengths, E, H, max_len=0):
    g = torch.Generator().manual_seed(seed)
    N = int(sum(lengths))
    q, k, v = (torch.randn(N, E, generator=g, dtype=torch.float64) for _ in range(3))
    dout = torch.randn(len(lengths), E, generator=g, dtype=torch.float64)
    return q, k, v, _offsets(lengths), dout


def _attn_float64(q, k, v, off, H, max_len, dout):
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    out = R.self_attn_pool(*leaves, off, H, max_len)
    out.backward(dout)
    return out.detach(), [t.grad for t in leaves]


def _attn_shim(L, q, k, v, off, H, max_len, dout, grid=None):
    s = ShimSeq(L, grid)
    pooled, lse = s.self_attn_pool_fwd(q, k, v, off, H, max_len)
    return pooled, lse, s.self_attn_pool_bwd(q, k, v, off, H, max_len, lse, dout.float())


# (lengths, E, H, max_len, grid)
ATTN_CASES = {
    "empty_batch": ([], 16, 4, 0, 1),
    "all_zero_lengths": ([0, 0, 0], 16, 4, 0, 2),
    "length_one": ([1, 1, 0, 1], 8, 2, 0, 3),
    "several_key_tiles": ([130, 3, 64, 65, 0], 16, 4, 0, 2),
    "crop": ([7, 2, 0, 5, 3], 12, 3, 3, 2),
    "crop_across_tiles": ([150, 70], 8, 1, 66, 1),
    "one_head": ([9, 4, 0, 1], 32, 1, 0, 3),
    "eight_heads": ([11, 0, 6], 64, 8, 0, 4),
    "hd_1": ([5, 0, 3, 1], 4, 4, 0, 2),
    "hd_128": ([70, 9, 0], 256, 2, 0, 2),
    "hd_17": ([12, 3], 34, 2, 0, 1),
}


@pytest.mark.parametrize("tag", list(ATTN_CASES))
def test_attention_kernel_source_against_float64(kern, tag):
    """pooled, dq, dk and dv of both kernels against the float64 jagged restatement over the cover's corners: an empty
    batch, all lengths 0, length 1, lengths across several 64-row key tiles, a crop (also across tiles), H 1 and 8, hd
    1, 17 and 128; cropped rows get zero gradients."""
    lengths, E, H, mx, grid = ATTN_CASES[tag]
    q, k, v, off, dout = _attn_case(len(tag), lengths, E, H, mx)
    out_r, (dq_r, dk_r, dv_r) = _attn_float64(q, k, v, off, H, mx, dout)
    pooled, lse, (dq, dk, dv) = _attn_shim(kern, q, k, v, off, H, mx, dout, grid)
    _close(_np(pooled), out_r, 1e-5, "pooled")
    for got, want, nm in ((dq, dq_r, "dq"), (dk, dk_r, "dk"), (dv, dv_r, "dv")):
        _close(_np(got), want, 2e-5, nm)
    assert torch.isfinite(lse).all()
    if mx > 0:
        lens = off[1:] - off[:-1]
        for b in range(len(lengths)):
            rows = slice(int(off[b]) + min(int(lens[b]), mx), int(off[b + 1]))
            assert float(dq[rows].abs().sum() + dk[rows].abs().sum() + dv[rows].abs().sum()) == 0


@pytest.mark.parametrize("grid", [1, 5])
def test_attention_kernel_source_reruns_bit_identical(kern, grid):
    """Reruns give identical bits, and so do different grids: every (sample, head) item owns its outputs."""
    q, k, v, off, dout = _attn_case(3, [20, 0, 70, 1, 9], 16, 4)
    a = _attn_shim(kern, q, k, v, off, 4, 0, dout, grid)
    b = _attn_shim(kern, q, k, v, off, 4, 0, dout, grid)
    c = _attn_shim(kern, q, k, v, off, 4, 0, dout, 2)
    for x, y, z in zip(torch.utils._pytree.tree_leaves(a), torch.utils._pytree.tree_leaves(b),
                       torch.utils._pytree.tree_leaves(c)):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_attention_kernel_source_refuses_outside_cover(kern):
    q, k, v, off, _ = _attn_case(1, [3, 2], 16, 4)
    f = [t.float() for t in (q, k, v)]

    def args(**kw):
        a = ShimSeq.args(*f, off, 4, 0)
        a.pooled = a.lse = 1
        for key, val in kw.items():
            setattr(a, key, val)
        return a

    assert kern.seq_attn_check(ctypes.byref(args()), 0) == 0
    assert kern.seq_attn_check(ctypes.byref(args()), 1) == 1            # no gradient buffers
    for kw in (dict(hd=129), dict(hd=0), dict(H=0), dict(max_len=-1), dict(ldq=15), dict(pooled=None)):
        assert kern.seq_attn_check(ctypes.byref(args(**kw)), 0) == 1, kw


@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("max_len", [0, 3])
def test_pool_kernel_source_against_float64(kern, mean, max_len):
    lengths = [0, 1, 5, 2, 9, 3, 0, 4, 12]
    g = torch.Generator().manual_seed(7)
    seq = torch.randn(sum(lengths), 20, generator=g, dtype=torch.float64)
    off = _offsets(lengths)
    dout = torch.randn(len(lengths), 20, generator=g, dtype=torch.float64)
    leaf = seq.clone().requires_grad_(True)
    want = R.pooling_encoder(leaf, off, max_len, mean)
    want.backward(dout)
    s = ShimSeq(kern)
    _close(_np(s.jagged_pool_fwd(seq, off, max_len, mean)), want.detach(), 1e-6, "out")
    _close(_np(s.jagged_pool_bwd(dout, off, seq.shape[0], max_len, mean)), leaf.grad, 1e-6, "d_seq")
    empty = torch.zeros(1, dtype=torch.int64)
    assert s.jagged_pool_fwd(seq[:0], empty, max_len, mean).shape == (0, 20)


# ---- the restatement and this repo's encoders against the reference's own -------------------------------------------
SA_TAGS = sorted({k[3:-len("_keys")] for k in GOLD.files if k.startswith("sa_") and k.endswith("_keys")})
POOL_TAGS = ["sum", "mean", "sum_crop", "mean_crop"]


def test_fixture_covers_the_issue_cases():
    assert set(SA_TAGS) == {"ref_test", "default", "one_head", "hd_1", "crop", "equal", "equal_crop"}
    lens = np.concatenate([GOLD[f"sa_{t}_lengths"] for t in SA_TAGS])
    assert {0, 1}.issubset(set(lens.tolist())) and lens.max() > 64
    assert GOLD["sa_ref_test_seq"].shape[1] > GOLD["sa_ref_test_lengths"].max()
    assert [int(x) for x in GOLD["sa_default_shape"]][1:3] == [512, 8]
    for t in SA_TAGS:                 # mixed lengths: the reference's gradients are NaN; equal lengths: stored
        assert bool(GOLD[f"sa_{t}_grads_nan"]) == (f"sa_{t}_dseq" not in GOLD.files)
    assert bool(GOLD["sa_crop_grads_nan"]) and not bool(GOLD["sa_equal_crop_grads_nan"])


def _sa_encoder(tag):
    """This repo's encoder from the reference's initialisation (torch.manual_seed(0)), pinned by the stored sums."""
    D, E, H, mx = (int(x) for x in GOLD[f"sa_{tag}_shape"])
    torch.manual_seed(0)
    enc = SelfAttentionEncoder(D, "seq", E, num_heads=H, max_seq_length=mx)
    assert list(enc.state_dict()) == list(GOLD[f"sa_{tag}_keys"])
    for k, v in enc.state_dict().items():
        np.testing.assert_allclose(float(v.double().sum()), float(GOLD[f"sa_{tag}_sum__{k}"]), rtol=1e-12, atol=1e-9)
    return enc, H, mx


def _jagged(tag, pre=None):
    pre = pre or f"sa_{tag}_"
    lengths = GOLD[pre + "lengths"]
    seqp = GOLD[pre + "seq"]
    rows = np.concatenate([seqp[b, :n] for b, n in enumerate(lengths)] + [np.zeros((0, seqp.shape[2]))])
    return lengths, _offsets(lengths), rows


def _rows_of(padded, lengths):
    return np.concatenate([padded[b, :n] for b, n in enumerate(lengths)] + [np.zeros((0, padded.shape[2]))])


@pytest.mark.parametrize("tag", SA_TAGS)
def test_padded_path_is_the_reference(tag):
    """TZK_DIN_JAGGED=0: the padded formulation reproduces the reference's output, and its gradients where they are
    finite; where lengths differ it gives the same NaN gradients."""
    enc, _, _ = _sa_encoder(tag)
    enc = enc.double()
    pre = f"sa_{tag}_"
    seq = torch.from_numpy(GOLD[pre + "seq"]).requires_grad_(True)
    out = enc({"seq.sequence": seq, "seq.sequence_length": torch.from_numpy(GOLD[pre + "lengths"])})
    np.testing.assert_allclose(out.detach().numpy(), GOLD[pre + "out"], rtol=1e-10, atol=1e-10)
    out.backward(torch.from_numpy(GOLD[pre + "dout"]))
    if bool(GOLD[pre + "grads_nan"]):
        assert any(bool(torch.isnan(p.grad).any()) for p in enc.parameters())
        return
    np.testing.assert_allclose(seq.grad.numpy(), GOLD[pre + "dseq"], rtol=1e-9, atol=1e-9)
    for k, p in enc.named_parameters():
        np.testing.assert_allclose(p.grad.numpy(), GOLD[pre + "grad__" + k], rtol=1e-9, atol=1e-9, err_msg=k)


def _restatement(tag, enc, H, mx):
    lengths, off, rows = _jagged(tag)
    params = {k: v.detach().double() for k, v in enc.state_dict().items()}
    for v in params.values():
        v.requires_grad_(True)
    seq = torch.from_numpy(rows).requires_grad_(True)
    out = R.self_attention_encoder(seq, off, params, H, mx)
    out.backward(torch.from_numpy(GOLD[f"sa_{tag}_dout"]))
    return out.detach(), seq.grad, {k: v.grad for k, v in params.items()}


@pytest.mark.parametrize("tag", SA_TAGS)
def test_restatement_matches_fixture_with_finite_gradients(tag):
    enc, H, mx = _sa_encoder(tag)
    out, dseq, grads = _restatement(tag, enc, H, mx)
    np.testing.assert_allclose(out.numpy(), GOLD[f"sa_{tag}_out"], rtol=1e-10, atol=1e-10)
    assert torch.isfinite(dseq).all() and all(torch.isfinite(g).all() for g in grads.values())
    if not bool(GOLD[f"sa_{tag}_grads_nan"]):
        lengths = GOLD[f"sa_{tag}_lengths"]
        np.testing.assert_allclose(dseq.numpy(), _rows_of(GOLD[f"sa_{tag}_dseq"], lengths), rtol=1e-9, atol=1e-9)
        for k, g in grads.items():
            np.testing.assert_allclose(g.numpy(), GOLD[f"sa_{tag}_grad__{k}"], rtol=1e-9, atol=1e-9, err_msg=k)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", SA_TAGS)
def test_jagged_encoder_matches_fixture_and_restatement(kern, tag, fused):
    """The encoder over jagged rows in float32, on the torch path and on the fused path (host build of the kernels):
    the reference's output on every case, its gradients where they are finite, and the float64 restatement's finite
    gradients everywhere."""
    if fused and tag == "default":
        pytest.skip("E 512 runs on the GPU tests; the host emulation of 48 CTAs x 256 threads is slow")
    enc, H, mx = _sa_encoder(tag)
    _, want_dseq, want_grads = _restatement(tag, enc, H, mx)
    lengths, off, rows = _jagged(tag)
    seq = torch.from_numpy(rows).float().requires_grad_(True)
    emb = {"seq.sequence": seq, "seq.sequence_length": torch.from_numpy(lengths), "seq.sequence_offsets": off}
    be = ShimBackend(kern) if fused else MetricOracleKernels()
    with Fn.use_backend(be):
        out = enc(emb)
        out.backward(torch.from_numpy(GOLD[f"sa_{tag}_dout"]).float())
    assert be.seq.attn_calls == 2 if fused else True
    _close(_np(out), GOLD[f"sa_{tag}_out"], 2e-5, "out")
    _close(_np(seq.grad), want_dseq, 5e-5, "d_seq")
    for k, p in enc.named_parameters():
        _close(_np(p.grad), want_grads[k], 5e-5, k)


def test_fused_path_refused_outside_cover_takes_torch(kern):
    """hd 160 is outside the cover; dropout in training cannot match torch's RNG: both take the torch path."""
    be = ShimBackend(kern)
    q = torch.zeros(3, 160)
    with Fn.use_backend(be):
        assert Fn.self_attn_pool_usable(q, 2, 0.0, True)
        assert not Fn.self_attn_pool_usable(q, 1, 0.0, True)
        assert not Fn.self_attn_pool_usable(q, 2, 0.1, True) and Fn.self_attn_pool_usable(q, 2, 0.1, False)
        assert not Fn.self_attn_pool_usable(q.double(), 2, 0.0, True)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert not Fn.self_attn_pool_usable(q, 2, 0.0, True)
        torch.manual_seed(0)
        enc = SelfAttentionEncoder(8, "seq", 160, num_heads=1)
        lengths = [3, 0, 2]
        seq = torch.randn(5, 8)
        out = enc({"seq.sequence": seq, "seq.sequence_length": torch.tensor(lengths),
                   "seq.sequence_offsets": _offsets(lengths)})
        out.sum().backward()
    assert be.seq.attn_calls == 0 and all(torch.isfinite(p.grad).all() for p in enc.parameters())
    assert not Fn.self_attn_pool_usable(q, 2, 0.0, True)           # no backend: CPU tensors never take the kernels


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tag", POOL_TAGS)
def test_pooling_encoder_matches_fixture(kern, tag, fused):
    kind, mx = {"sum": ("sum", 0), "mean": ("mean", 0), "sum_crop": ("sum", 3), "mean_crop": ("mean", 3)}[tag]
    enc = PoolingEncoder(8, "seq", pooling_type=kind, max_seq_length=mx)
    lengths, off, rows = _jagged(tag, "pool_")
    seq = torch.from_numpy(rows).float().requires_grad_(True)
    be = ShimBackend(kern) if fused else MetricOracleKernels()
    with Fn.use_backend(be):
        out = enc({"seq.sequence": seq, "seq.sequence_length": torch.from_numpy(lengths),
                   "seq.sequence_offsets": off})
        out.backward(torch.from_numpy(GOLD["pool_dout"]).float())
    assert be.seq.pool_calls == 2 if fused else True
    _close(_np(out), GOLD[f"pool_{tag}_out"], 1e-6, "out")
    _close(_np(seq.grad), _rows_of(GOLD[f"pool_{tag}_dseq"], lengths), 1e-6, "d_seq")
    padded = PoolingEncoder(8, "seq", pooling_type=kind, max_seq_length=mx)(
        {"seq.sequence": torch.from_numpy(GOLD["pool_seq"]), "seq.sequence_length": torch.from_numpy(lengths)})
    np.testing.assert_allclose(padded.numpy(), GOLD[f"pool_{tag}_out"], rtol=1e-12, atol=1e-12)


# ---- schemas, factory and configs ------------------------------------------------------------------------------------
def _encoder_cfg(body):
    return parse_text("model_config { feature_groups { group_name: \"all\" sequence_encoders { " + body + " } } }"
                      ).model_config.feature_groups[0].sequence_encoders[0]


def test_schema_defaults_and_factory():
    dims = {"s.sequence": 48, "s.query": 48}
    sa = _encoder_cfg('self_attention_encoder { input: "s" }')
    c = sa.self_attention_encoder
    assert (c.multihead_attn_dim, c.num_heads, c.dropout, c.max_seq_length) == (512, 8, 0.0, 0)
    enc = _create_seq_encoder(sa, dims)
    assert isinstance(enc, SelfAttentionEncoder) and enc.output_dim() == 512
    assert list(enc.state_dict()) == list(GOLD["sa_default_keys"])
    pc = _encoder_cfg('pooling_encoder { input: "s" }')
    assert (pc.pooling_encoder.pooling_type, pc.pooling_encoder.max_seq_length) == ("mean", 0)
    assert isinstance(_create_seq_encoder(pc, dims), PoolingEncoder)
    mw = _encoder_cfg('multi_window_din_encoder { input: "s" windows_len: [1, 2] attn_mlp { hidden_units: [4] } }')
    assert mw.multi_window_din_encoder.attn_mlp.activation == "nn.ReLU"
    assert _create_seq_encoder(mw, dims).output_dim() == 48 * 3
    with pytest.raises(AssertionError, match="sum\\|mean"):
        _create_seq_encoder(_encoder_cfg('pooling_encoder { input: "s" pooling_type: "max" }'), dims)
    with pytest.raises(AssertionError, match="divisible"):
        _create_seq_encoder(_encoder_cfg('self_attention_encoder { input: "s" multihead_attn_dim: 10 num_heads: 3 }'),
                            dims)
    with pytest.raises(NotImplementedError, match="simple_attention"):
        _create_seq_encoder(_encoder_cfg('simple_attention { input: "s" }'), dims)


def test_multi_window_din_encoder_in_a_deep_group_equals_the_tdm_fixture():
    """The factory's multi_window_din_encoder is TDM's encoder: the TDM fixture's encoder case through it."""
    gold = np.load(os.path.join(HERE, "golden", "ref_tdm.npz"))
    pre = "enc_w125_relu84_"
    C, Dq = gold[pre + "seq"].shape[2], gold[pre + "query"].shape[1]
    windows = ", ".join(str(int(w)) for w in gold[pre + "windows"])
    hidden = ", ".join(str(int(h)) for h in gold[pre + "hidden"])
    cfg = _encoder_cfg(f'multi_window_din_encoder {{ input: "seq" windows_len: [{windows}] attn_mlp {{ '
                       f'hidden_units: [{hidden}] activation: "{gold[pre + "act"]}" }} }}')
    enc = _create_seq_encoder(cfg, {"seq.sequence": C, "seq.query": Dq})
    enc.load_state_dict({k: torch.from_numpy(gold[pre + "sd__" + k]).to(v.dtype) for k, v in enc.state_dict().items()})
    enc = enc.double()
    out = enc({"seq.query": torch.from_numpy(gold[pre + "query"]), "seq.sequence": torch.from_numpy(gold[pre + "seq"]),
               "seq.sequence_length": torch.from_numpy(gold[pre + "lengths"])})
    np.testing.assert_allclose(out.detach().numpy(), gold[pre + "out"], rtol=1e-10, atol=1e-10)


def test_seq_encoders_config_parses_and_is_edited():
    assert "dbmtl_taobao_seq_encoders" in EDITED_GENERATORS and "dbmtl_taobao_seq_encoders" in BUILTINS
    cfg = parse_text(EDITED_GENERATORS["dbmtl_taobao_seq_encoders"]())
    encs = cfg.model_config.feature_groups[0].sequence_encoders
    assert [e.WhichOneof("seq_module") for e in encs] == ["din_encoder", "self_attention_encoder", "pooling_encoder"]
    assert encs[1].self_attention_encoder.multihead_attn_dim == 512 and encs[2].pooling_encoder.pooling_type == "mean"
    assert "self_attention_encoder" in EDITED_GENERATORS["dbmtl_taobao_seq_encoders"].__doc__


@pytest.fixture(scope="module")
def seq_pipe():
    return Pipeline("dbmtl_taobao_seq_encoders", device="cpu", max_rows=200, seed=3, capturable=False)


def test_seq_encoders_config_trains_on_the_fused_path_and_evaluates(kern, seq_pipe):
    pipe = seq_pipe
    eg = pipe.model.embedding_group
    assert eg.group_total_dim("all") == 16 * 16 + 48 + 512 + 48
    assert [type(e).__name__ for e in eg._group_name_to_seq_encoders["all"]] == \
        ["DINEncoder", "SelfAttentionEncoder", "PoolingEncoder"]
    batch = pipe.synthetic_batch(24, seed=1)
    be = ShimBackend(kern, grid=8)
    with Fn.use_backend(be):
        ls = [float(pipe.eager_step(batch)) for _ in range(2)]
        m = pipe.evaluate([pipe.synthetic_batch(24, seed=s) for s in range(2)])
    assert np.isfinite(ls).all() and ls[1] < ls[0]
    assert be.seq.attn_calls == 2 * 2 + 2 and be.seq.pool_calls == 2 * 2 + 2
    assert all(np.isfinite(v) for v in m.values())


def test_seq_encoders_config_jagged_and_padded_forwards_agree(monkeypatch):
    from oracle_backend import OracleKernels

    outs = []
    for jagged in ("1", "0"):
        monkeypatch.setenv("TZK_DIN_JAGGED", jagged)
        pipe = Pipeline("dbmtl_taobao_seq_encoders", device="cpu", max_rows=200, seed=3, capturable=False)
        jag = any(getattr(impl, "_jagged_for_attention", None) for impl in pipe.model.embedding_group.seq_emb_impls.values())
        assert jag == (jagged == "1")
        pipe.model.eval()
        with Fn.use_backend(OracleKernels()), torch.no_grad():
            preds = pipe.model.predict(pipe.synthetic_batch(24, seed=1))
        outs.append({k: v.clone() for k, v in preds.items()})
    for k in outs[0]:
        torch.testing.assert_close(outs[0][k], outs[1][k], rtol=2e-5, atol=2e-6)


def test_seq_encoders_two_ranks_equal_the_unsharded_twin():
    """dbmtl_taobao_seq_encoders over gloo W = 2 against the unsharded model on the concatenated batch."""
    from test_distributed_cpu import _run

    _run(2, "dbmtl_taobao_seq_encoders", "mixed", rw_min_rows=250)
