"""train_config.mixed_precision on the CPU: the config mapping, the DLRM glue under bf16 autocast against a fixture made
by the reference's own modules, the BF16 interaction kernels' SOURCE against a float64 restatement, and CPU train steps
of the reference example configs with "BF16".

Rounding-point bounds used for the kernels (bf16: 8 significant bits; ulp(v) = 2^(floor(log2|v|) - 7)):
  * A value the kernel rounds to bf16 from an fp32 sum of n = 16 or 32 exact bf16 products differs from the exact sum by
    at most the fp32 accumulation error, bounded by 2 n 2^-24 sum|products| (twice the textbook gamma_n, to leave room
    for the tensor cores' unspecified internal order); rounding both to bf16 then moves them at most one ulp apart.  So
    |kernel - bf16(exact)| <= ulp + 2^-19 sum|products| for the forward pairs (n = 16) and e_i = ulp + 2^-18
    sum|products| for the backward products g1 = bf16(G F), g2 = bf16(G^T F) (n = 32).
  * d_sparse = fp32(fp32(g1 + g2) + dX): two fp32 roundings of at most 2^-24 relative each, so
    |kernel - ref| <= e1 + e2 + 2^-23 (|g1| + |g2| + |dX|).
  * d_dense = bf16(bf16(fp32(g1 + g2)) + dX): each bf16 rounding adds at most one ulp of its result to the difference
    carried in, so |kernel - ref| <= e1 + e2 + 2^-23 (|s| + |dX|) + 2 ulp(s) + 2 ulp(d_dense).
"""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
EXP = os.path.join(HERE, "native")
REF_EXAMPLES = os.path.join(HERE, "golden", "ref_examples")
GOLD = np.load(os.path.join(HERE, "golden", "ref_dlrm_bf16.npz"))
P, I32, I64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
N, D, PAIRS, ROW = 27, 16, 351, 784
IU = np.triu_indices(N, 1)


# ---------------------------------------------------------------------------------------------------- bf16 helpers
def bf16_bits(x):
    """fp32 -> bf16 bit pattern, round to nearest even."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bits_f(h):
    return (h.astype(np.uint32) << 16).view(np.float32)


def bf16_of(x):
    """float64 -> the nearest bf16 value (ties to even), as float64: one rounding, no detour through fp32."""
    m, e = np.frexp(np.asarray(x, dtype=np.float64))
    return np.ldexp(np.rint(m * 256.0), e - 8)


def ulp(v):
    a = np.abs(np.asarray(v, dtype=np.float64))
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    return np.where(a > 0, np.ldexp(1.0, (e - 7).astype(np.int64)), 2.0 ** -133)


def fwd_reference(dense_bits, sparse):
    """(pairs as bf16(exact) float64, their bound, copied columns as bit patterns)."""
    B = sparse.shape[0]
    Fm = np.concatenate([bits_f(dense_bits)[:, None, :], bits_f(bf16_bits(sparse)).reshape(B, 26, D)], axis=1)
    Fm = Fm.astype(np.float64)
    Z = Fm @ Fm.transpose(0, 2, 1)
    A = np.abs(Fm) @ np.abs(Fm).transpose(0, 2, 1)
    ref = bf16_of(Z[:, IU[0], IU[1]])
    return ref, A[:, IU[0], IU[1]], np.concatenate([dense_bits, bf16_bits(sparse)], axis=1)


def check_fwd(out_bits, dense_bits, sparse, exact_share=None):
    ref, A, copied = fwd_reference(dense_bits, sparse)
    got = bits_f(out_bits[:, :PAIRS]).astype(np.float64)
    bound = ulp(np.maximum(np.abs(ref), np.abs(got))) + 2.0 ** -19 * A
    assert np.all(np.abs(got - ref) <= bound), np.max(np.abs(got - ref) / bound)
    assert np.all(out_bits[:, PAIRS] == 0)
    np.testing.assert_array_equal(out_bits[:, 352:ROW], copied)
    if exact_share is not None:
        assert np.mean(got == ref) >= exact_share


def bwd_reference(d_out_bits, dense_bits, sparse):
    B = sparse.shape[0]
    Fm = np.concatenate([bits_f(dense_bits)[:, None, :], bits_f(bf16_bits(sparse)).reshape(B, 26, D)], axis=1)
    Fm = Fm.astype(np.float64)
    G = np.zeros((B, N, N))
    G[:, IU[0], IU[1]] = bits_f(d_out_bits[:, :PAIRS])
    r1, r2 = bf16_of(G @ Fm), bf16_of(G.transpose(0, 2, 1) @ Fm)
    e1 = ulp(r1) + 2.0 ** -18 * (np.abs(G) @ np.abs(Fm))
    e2 = ulp(r2) + 2.0 ** -18 * (np.abs(G.transpose(0, 2, 1)) @ np.abs(Fm))
    s = (r1.astype(np.float32) + r2.astype(np.float32)).astype(np.float32)
    dx = bits_f(d_out_bits[:, 352:ROW]).reshape(B, N, D)
    dd = bits_f(bf16_bits((bits_f(bf16_bits(s[:, 0])) + dx[:, 0]).astype(np.float32))).astype(np.float64)
    ds = (s[:, 1:] + dx[:, 1:]).astype(np.float32).reshape(B, -1).astype(np.float64)
    b_ds = (e1 + e2 + 2.0 ** -23 * (np.abs(r1) + np.abs(r2) + np.abs(dx)))[:, 1:].reshape(B, -1)
    b_dd = (e1 + e2)[:, 0] + 2.0 ** -23 * (np.abs(s[:, 0]) + np.abs(dx[:, 0])) + 2 * ulp(s[:, 0]) + 2 * ulp(dd)
    return dd, b_dd, ds, b_ds


def check_bwd(d_dense_bits, d_sparse, d_out_bits, dense_bits, sparse, exact_share=None):
    dd, b_dd, ds, b_ds = bwd_reference(d_out_bits, dense_bits, sparse)
    got_dd = bits_f(d_dense_bits).astype(np.float64)
    got_ds = d_sparse.astype(np.float64)
    assert np.all(np.abs(got_dd - dd) <= b_dd), np.max(np.abs(got_dd - dd) / b_dd)
    assert np.all(np.abs(got_ds - ds) <= b_ds), np.max(np.abs(got_ds - ds) / b_ds)
    if exact_share is not None:
        assert np.mean(got_dd == dd) >= exact_share and np.mean(got_ds == ds) >= exact_share


def inputs(B, seed, pad=0):
    rng = np.random.default_rng(seed)
    dense = np.zeros((B, D + pad), np.uint16)
    dense[:, :D] = bf16_bits(rng.standard_normal((B, D)))
    sparse = np.zeros((B, 26 * D + pad), np.float32)
    sparse[:, :26 * D] = rng.standard_normal((B, 26 * D))
    d_out = np.zeros((B, ROW + 8 * (pad > 0)), np.uint16)
    d_out[:, :ROW] = bf16_bits(rng.standard_normal((B, ROW)))
    d_out[:, PAIRS] = 0
    return dense, sparse, d_out


# ---------------------------------------------------------------------------------------------------- config mapping
def test_mixed_precision_mapping():
    from torcheasyrec_b200.rank_models import mixed_precision_to_dtype

    assert mixed_precision_to_dtype("BF16") is torch.bfloat16
    assert mixed_precision_to_dtype("FP16") is torch.float16
    assert mixed_precision_to_dtype("") is None and mixed_precision_to_dtype(None) is None
    with pytest.raises(ValueError, match="Unknown mixed_precision"):
        mixed_precision_to_dtype("bf16")


def test_pipeline_honours_mixed_precision_and_refuses_grad_scaler():
    from torcheasyrec_b200.engine import Pipeline

    assert Pipeline("dlrm_criteo", device="cpu", max_rows=50).train_wrapper.mixed_dtype is None
    p = Pipeline("dlrm_criteo", device="cpu", max_rows=50, edits={"train_config.mixed_precision": "BF16"})
    assert p.train_wrapper.mixed_dtype is torch.bfloat16 and p.train_wrapper.device_type == "cpu"
    with pytest.raises(ValueError):
        Pipeline("dlrm_criteo", device="cpu", max_rows=50, edits={"train_config.mixed_precision": "INT8"})
    with pytest.raises(NotImplementedError, match="grad_scaler"):
        Pipeline("dlrm_criteo", device="cpu", max_rows=50,
                 edits={"train_config.mixed_precision": "BF16", "train_config.grad_scaler.init_scale": 1024.0})
    # a grad_scaler block without mixed_precision is accepted and leaves the step in fp32, as before
    assert Pipeline("dlrm_criteo", device="cpu", max_rows=50,
                    edits={"train_config.grad_scaler.init_scale": 1024.0}).train_wrapper.mixed_dtype is None


# ---------------------------------------------------------------------------------------------------- golden fixture
def test_dlrm_bf16_glue_reproduces_reference_autocast():
    """The repo's DLRM-Criteo step on the CPU (oracle backend for the sparse side) with mixed_precision "BF16", fed the
    fixture's dense input and pooled embeddings, runs the same torch ops as the reference under autocast: logits, loss,
    the pooled-embedding gradient and every dense parameter gradient are bit-identical."""
    from oracle_backend import OracleKernels

    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.engine import Pipeline

    pipe = Pipeline("dlrm_criteo", device="cpu", max_rows=50, seed=1, edits={"train_config.mixed_precision": "BF16"})
    m = pipe.model
    sd = {k[4:]: torch.from_numpy(v) for k, v in GOLD.items() if k.startswith("sd__")}
    missing = m.load_state_dict(sd, strict=False)
    assert not missing.unexpected_keys
    sparse = torch.from_numpy(GOLD["sparse"]).requires_grad_()
    dense_in = torch.from_numpy(GOLD["dense_in"])
    m._dense_group_input = lambda batch: dense_in
    m.build_input = lambda batch: {m._sparse_group_name: sparse}
    batch = types.SimpleNamespace(labels={m._label_name: torch.from_numpy(GOLD["labels"])})
    with Fn.use_backend(OracleKernels()):
        total, (_, preds, _) = pipe.train_wrapper(batch)
        total.backward()
    assert preds["logits"].dtype == torch.bfloat16 and total.dtype == torch.float32
    np.testing.assert_array_equal(preds["logits"].float().numpy(), GOLD["logits"])
    np.testing.assert_array_equal(total.detach().numpy(), GOLD["loss"])
    np.testing.assert_array_equal(sparse.grad.numpy(), GOLD["dsparse"])
    params = dict(m.named_parameters())
    for k in GOLD:
        if k.startswith("grad__"):
            np.testing.assert_array_equal(params[k[6:]].grad.numpy(), GOLD[k], err_msg=k)


# ---------------------------------------------------------------------------------------------------- kernel source
@pytest.fixture(scope="module")
def ib16(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("shim") / "libib16_cpu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-DTZK_CPU_SHIM", "-Wno-unknown-pragmas", "-I", EXP, "-x", "c++",
                    os.path.join(EXP, "interact_bf16_standalone.cu"), "-shared", "-fPIC", "-o", out], check=True)
    L = ctypes.CDLL(out)
    L.tzk_ib16_fwd.argtypes = [P, I64, P, I64, I64, P, I64, I32]
    L.tzk_ib16_bwd.argtypes = [P, I64, P, I64, P, I64, I64, P, I64, P, I64, I32]
    return L


CASES = [(1, 1, 0), (31, 1, 0), (32, 1, 4), (33, 2, 0), (200, 3, 4)]      # (B, grid, row padding)


@pytest.mark.parametrize("B,grid,pad", CASES)
def test_bf16_forward_source_matches_float64(ib16, B, grid, pad):
    dense, sparse, _ = inputs(B, 100 + B, pad)
    ld_out = ROW + 8 * (pad > 0)
    out = np.full((B, ld_out), 0xFFFF, dtype=np.uint16)
    ib16.tzk_ib16_fwd(dense.ctypes.data, D + pad, sparse.ctypes.data, 26 * D + pad, B, out.ctypes.data, ld_out, grid)
    check_fwd(out[:, :ROW], dense[:, :D], sparse[:, :26 * D], exact_share=0.98)
    if pad:
        assert np.all(out[:, ROW:] == 0xFFFF)


@pytest.mark.parametrize("B,grid,pad", CASES)
def test_bf16_backward_source_matches_float64(ib16, B, grid, pad):
    dense, sparse, d_out = inputs(B, 200 + B, pad)
    d_dense = np.full((B, D + pad), 0xFFFF, dtype=np.uint16)
    d_sparse = np.full((B, 26 * D + pad), np.nan, dtype=np.float32)
    ib16.tzk_ib16_bwd(d_out.ctypes.data, d_out.shape[1], dense.ctypes.data, D + pad, sparse.ctypes.data, 26 * D + pad, B,
                      d_dense.ctypes.data, D + pad, d_sparse.ctypes.data, 26 * D + pad, grid)
    check_bwd(d_dense[:, :D], d_sparse[:, :26 * D], d_out[:, :ROW], dense[:, :D], sparse[:, :26 * D], exact_share=0.98)
    if pad:
        assert np.all(d_dense[:, D:] == 0xFFFF) and np.isnan(d_sparse[:, 26 * D:]).all()


def test_bwd_restatement_matches_torch_autocast():
    """The float64 restatement's rounding points are torch's: autograd through the reference's bmm + triu + cat under
    CPU bf16 autocast gives the same d_dense and d_sparse bits (exact-sum products: small-integer inputs)."""
    rng = np.random.default_rng(5)
    B = 6
    dense_f = rng.integers(-3, 4, (B, D)).astype(np.float32)
    sparse_np = rng.integers(-3, 4, (B, 26 * D)).astype(np.float32)
    dX = bits_f(bf16_bits(rng.standard_normal((B, 783)).astype(np.float32)))
    dense = torch.from_numpy(dense_f).to(torch.bfloat16).requires_grad_()
    sparse = torch.from_numpy(sparse_np).requires_grad_()
    with torch.autocast("cpu", torch.bfloat16):
        feat = torch.cat([dense.unsqueeze(1), sparse.reshape(B, 26, D)], dim=1)
        z = torch.bmm(feat, feat.transpose(1, 2))[:, IU[0], IU[1]]
        x = torch.cat([torch.cat([z, dense], dim=-1), sparse], dim=-1)
    x.backward(torch.from_numpy(dX))
    d_out = np.zeros((B, ROW), np.uint16)
    d_out[:, :PAIRS] = bf16_bits(dX[:, :PAIRS])
    d_out[:, 352:] = bf16_bits(dX[:, PAIRS:])
    dd, _, ds, _ = bwd_reference(d_out, bf16_bits(dense_f), sparse_np)
    np.testing.assert_array_equal(dense.grad.float().numpy(), dd)
    np.testing.assert_array_equal(sparse.grad.numpy(), ds)


# ---------------------------------------------------------------------------------------------------- example configs
@pytest.mark.parametrize("name", ["dlrm_criteo", "deepfm_criteo", "mmoe_taobao", "multi_tower_din_taobao"])
def test_reference_example_config_runs_with_bf16(name):
    """The reference's example config with mixed_precision "BF16": two CPU steps on the oracle; the loss is finite and
    moves."""
    from oracle_backend import OracleKernels

    from torcheasyrec_b200 import functional as Fn
    from torcheasyrec_b200.engine import Pipeline

    pipe = Pipeline(os.path.join(REF_EXAMPLES, name + ".config"), device="cpu", max_rows=200, seed=3,
                    edits={"train_config.mixed_precision": "BF16"})
    batch = pipe.synthetic_batch(24, seed=1)
    with Fn.use_backend(OracleKernels()):
        l0 = float(pipe.eager_step(batch))
        l1 = float(pipe.eager_step(batch))
    assert np.isfinite([l0, l1]).all()
    assert l1 != l0
