"""GPU parity: every tzk kernel (through the C-ABI) against the CPU oracle on seeded inputs.

Bars (BASELINE.json north_star): bit-exact for integer / index work; <= 1e-5 relative for pooled
embeddings, interactions and updated weights.
"""
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import tzk_oracle as O
from torcheasyrec_b200.kernels import ColPlan, build_layout

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_dense_modules.npz"))
DEV = "cuda"


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def random_kjt(rng, F, B, rows, max_len, empty_frac=0.2, fixed_len=None):
    if fixed_len is not None:
        lengths = np.full(F * B, fixed_len, dtype=np.int32)
    else:
        lengths = rng.integers(0, max_len + 1, size=F * B).astype(np.int32)
        lengths[rng.random(F * B) < empty_frac] = 0
    offsets = O.lengths_to_offsets(lengths)
    parts = [rng.integers(0, rows[f], size=int(lengths[f * B:(f + 1) * B].sum())) for f in range(F)]
    ids = np.concatenate(parts).astype(np.int64) if offsets[-1] else np.zeros(0, np.int64)
    return ids, lengths, offsets


def make_arena(lay, tables, feat_table):
    arena = np.zeros(lay.arena_elems, dtype=np.float32)
    seen = set()
    for f, t in enumerate(feat_table):
        if t in seen:
            continue
        seen.add(t)
        arena[lay.w_off[f]:lay.w_off[f] + tables[t].size] = tables[t].ravel()
    return arena


def split_arena(arena, lay, tables, feat_table):
    out = {}
    for f, t in enumerate(feat_table):
        out[t] = arena[lay.w_off[f]:lay.w_off[f] + tables[t].size].reshape(tables[t].shape)
    return [out[t] for t in range(len(tables))]


@pytest.mark.parametrize("n", [0, 1, 5, 4096, 4097, 100003, 26 * 65536])
def test_lengths_to_offsets_bit_exact(kernels, n):
    rng = np.random.default_rng(n)
    lengths = rng.integers(0, 9, size=n).astype(np.int32)
    got = kernels.lengths_to_offsets(cu(lengths)).cpu().numpy()
    np.testing.assert_array_equal(got, O.lengths_to_offsets(lengths))


@pytest.fixture(params=["general", "tile"])
def bwd_path(request, monkeypatch):
    """Both implementations of the gradient half of tzk_fused_bwd (csrc/tzk_bwd.cu): the general run kernels
    (default) and the shared-memory tile path (TZK_BWD_TILE=1)."""
    monkeypatch.setenv("TZK_BWD_TILE", "1" if request.param == "tile" else "0")
    return request.param


CASES = {
    # name: (rows, dims, feat_table, B, max_len)
    "criteo_like_L1": ([1000] * 6, [16] * 6, list(range(6)), 300, None),
    "deepfm_mixed_dims": ([50, 50, 700, 700], [4, 4, 16, 16], [0, 1, 2, 3], 257, 5),
    "shared_table": ([40, 900], [16, 8], [0, 1, 0, 1], 129, 4),
    "wide_rows": ([300, 20], [128, 64], [0, 1], 65, 3),
    "very_wide_rows": ([64], [256], [0], 33, 3),
    "unaligned_dims": ([30, 70], [13, 6], [0, 1], 77, 4),
    "tiny_tables_long_runs": ([3, 4, 10], [16, 16, 16], [0, 1, 2], 2000, 2),
    "multi_hot_33": ([5000], [16], [0], 50, 33),
    # tile path of the fused backward: runs that cross many tiles at the smallest (D=128 -> 32 positions) and the
    # largest (D=4 -> 1024 positions) tile size, next to short runs
    "long_runs_wide_rows": ([2, 300], [128, 128], [0, 1], 700, 2),
    "long_runs_d4": ([3, 20000], [4, 4], [0, 1], 3000, 2),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("pool", [O.POOL_SUM, O.POOL_MEAN])
def test_pooled_gather_fwd(kernels, case, pool):
    rows, dims, feat_table, B, max_len = CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()) % 1000)
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    F = len(feat_table)
    frows = [rows[t] for t in feat_table]
    ids, lengths, offsets = random_kjt(rng, F, B, frows, max_len or 1, fixed_len=1 if max_len is None else None)
    if len(ids) > 4:  # out-of-range ids read row 0 (A.9)
        ids[1] = frows[0] + 5 if lengths[:B].sum() > 1 else ids[1]
    lay = build_layout(rows, dims, feat_table, [pool] * F).to(DEV)
    arena = cu(make_arena(lay, tables, feat_table))
    got = kernels.pooled_gather_fwd(arena, lay, cu(ids), cu(offsets), B).cpu().numpy()
    want = O.pooled_lookup(tables, feat_table, [pool] * F, ids, offsets, B)
    if pool == O.POOL_SUM and (max_len is None):
        np.testing.assert_array_equal(got, want)  # L=1: pure copy, bit exact
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-7)


def test_pooled_gather_empty_batch_and_all_empty_bags(kernels):
    lay = build_layout([10], [16], [0], [0]).to(DEV)
    arena = torch.randn(lay.arena_elems, device=DEV)
    B = 8
    offsets = torch.zeros(B + 1, dtype=torch.int64, device=DEV)
    out = kernels.pooled_gather_fwd(arena, lay, torch.zeros(0, dtype=torch.int64, device=DEV), offsets, B)
    assert out.shape == (B, 16) and float(out.abs().sum()) == 0.0


def test_seq_gather_fwd(kernels):
    rng = np.random.default_rng(2)
    rows, dims, feat_table, B = [500, 60, 500], [16, 16, 16], [0, 1, 2], 40
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    ids, lengths, offsets = random_kjt(rng, 3, B, rows, 20)
    lay = build_layout(rows, dims, feat_table, [0] * 3).to(DEV)
    arena = cu(make_arena(lay, tables, feat_table))
    got = kernels.seq_gather_fwd(arena, lay, cu(ids), cu(offsets), B).cpu().numpy()
    np.testing.assert_array_equal(got, O.seq_lookup(tables, feat_table, ids, offsets, B))


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("opt", [O.OPT_SGD, O.OPT_ADAGRAD, O.OPT_ROWWISE_ADAGRAD])
@pytest.mark.parametrize("pool", [O.POOL_SUM, O.POOL_MEAN])
def test_fused_bwd(kernels, case, opt, pool, bwd_path):
    rows, dims, feat_table, B, max_len = CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()) % 1000 + 17)
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    F = len(feat_table)
    frows = [rows[t] for t in feat_table]
    ids, lengths, offsets = random_kjt(rng, F, B, frows, max_len or 1, fixed_len=1 if max_len is None else None)
    lay = build_layout(rows, dims, feat_table, [pool] * F).to(DEV)
    arena = cu(make_arena(lay, tables, feat_table))
    grad = rng.standard_normal((B, lay.total_dim)).astype(np.float32)
    lr, eps, gs = 0.05, 1e-8, 0.5
    if opt == O.OPT_ADAGRAD:
        st_np = [np.abs(rng.standard_normal(t.shape)).astype(np.float32) * 0.01 for t in tables]
        state = cu(make_arena(lay, st_np, feat_table))
    elif opt == O.OPT_ROWWISE_ADAGRAD:
        st_np = [np.abs(rng.standard_normal(t.shape[0])).astype(np.float32) * 0.01 for t in tables]
        state = cu(np.concatenate(st_np))
    else:
        st_np, state = [None] * len(tables), None
    two_steps = 2
    # Runs longer than 32 contributions are summed as 64 strided partials + a fixed tree (fbgemm's long-row
    # path is a tree too), the oracle adds sequentially: with ~700 cancelling terms per row both are ~1e-5
    # from the exact sum, and the accumulator s += g*g doubles the relative gap.  Weights stay within 1e-5.
    long_runs = case in ("tiny_tables_long_runs", "long_runs_wide_rows", "long_runs_d4")
    state_rtol = 3e-4 if long_runs else 2e-5
    w_rtol, w_atol = (5e-5, 5e-6) if long_runs else (1e-5, 1e-6)
    want = [t.copy() for t in tables]
    for _ in range(two_steps):  # second step exercises the updated state
        kernels.fused_bwd(opt, True, cu(grad), arena, state, lay, cu(ids), cu(offsets), B, lr, eps, gs)
        O.fused_update(opt, want, st_np, feat_table, [pool] * F, ids, offsets, B, grad, lr, eps, gs)
    got = split_arena(arena.cpu().numpy(), lay, tables, feat_table)
    for t in range(len(tables)):
        np.testing.assert_allclose(got[t], want[t], rtol=w_rtol, atol=w_atol, err_msg=f"table {t}")
    if opt == O.OPT_ADAGRAD:
        gs_ = split_arena(state.cpu().numpy(), lay, tables, feat_table)
        for t in range(len(tables)):
            np.testing.assert_allclose(gs_[t], st_np[t], rtol=state_rtol, atol=1e-7)
    if opt == O.OPT_ROWWISE_ADAGRAD:
        np.testing.assert_allclose(state.cpu().numpy(), np.concatenate(st_np), rtol=state_rtol, atol=1e-7)


def test_fused_bwd_is_run_to_run_deterministic(kernels, bwd_path):
    rng = np.random.default_rng(9)
    rows, dims, feat_table, B = [3, 7, 5000], [16, 16, 16], [0, 1, 2], 4096
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    ids, lengths, offsets = random_kjt(rng, 3, B, rows, 3)
    lay = build_layout(rows, dims, feat_table, [0] * 3).to(DEV)
    grad = cu(rng.standard_normal((B, lay.total_dim)).astype(np.float32))
    res = []
    for _ in range(3):
        arena = cu(make_arena(lay, tables, feat_table))
        state = torch.zeros_like(arena)
        kernels.fused_bwd(O.OPT_ADAGRAD, True, grad, arena, state, lay, cu(ids), cu(offsets), B, 0.01, 1e-8, 1.0)
        res.append(arena.cpu().numpy())
    np.testing.assert_array_equal(res[0], res[1])
    np.testing.assert_array_equal(res[0], res[2])


def test_fused_bwd_sequence_layout(kernels, bwd_path):
    rng = np.random.default_rng(21)
    rows, dims, feat_table, B = [400, 30, 400], [16, 16, 16], [0, 1, 2], 64
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    ids, lengths, offsets = random_kjt(rng, 3, B, rows, 12)
    lay = build_layout(rows, dims, feat_table, [0] * 3).to(DEV)
    arena = cu(make_arena(lay, tables, feat_table))
    state = torch.zeros_like(arena)
    grad = rng.standard_normal((len(ids), 16)).astype(np.float32)
    kernels.fused_bwd(O.OPT_ADAGRAD, False, cu(grad), arena, state, lay, cu(ids), cu(offsets), B, 0.02, 1e-8, 1.0)
    want = [t.copy() for t in tables]
    st = [np.zeros_like(t) for t in tables]
    O.fused_update(O.OPT_ADAGRAD, want, st, feat_table, [0] * 3, ids, offsets, B, grad, 0.02, 1e-8, 1.0, pooled=False)
    got = split_arena(arena.cpu().numpy(), lay, tables, feat_table)
    for t in range(3):
        np.testing.assert_allclose(got[t], want[t], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("W", [1, 2, 8])
@pytest.mark.parametrize("max_len", [None, 6])
def test_bucketize_rw_bit_exact(kernels, W, max_len):
    rng = np.random.default_rng(W * 10 + (max_len or 0))
    F, B = 5, 333
    rows = [39060, 3, 4, 100000, 17]  # hash_size % W != 0 and tables smaller than W (SURVEY §8c golden (5))
    ids, lengths, offsets = random_kjt(rng, F, B, rows, max_len or 1, fixed_len=1 if max_len is None else None)
    blocks = [O.rw_block_size(r, W) for r in rows]
    ol, oo, oi, op, inv = kernels.bucketize_rw(cu(ids), cu(offsets), F, B, W, cu(np.asarray(blocks, np.int64)),
                                               want_pos=True, want_inv=True)
    wl, wo, wi, wp = O.bucketize_rw(ids, offsets, F, B, W, blocks)
    np.testing.assert_array_equal(ol.cpu().numpy(), wl)
    np.testing.assert_array_equal(oo.cpu().numpy(), wo)
    np.testing.assert_array_equal(oi.cpu().numpy(), wi)
    np.testing.assert_array_equal(op.cpu().numpy(), wp)
    np.testing.assert_array_equal(inv.cpu().numpy()[wp], np.arange(len(wp)))


@pytest.mark.parametrize("W", [2, 8])
def test_bucketize_mixed_table_wise_and_row_wise(kernels, W):
    """table-wise features go whole to their owner; row-wise ones are split by block (cfg5-style mixed plan)."""
    rng = np.random.default_rng(W)
    F, B = 4, 200
    rows = [1000, 50, 77777, 9]
    ids, lengths, offsets = random_kjt(rng, F, B, rows, 4)
    blocks = [O.rw_block_size(rows[0], W), 1 << 62, O.rw_block_size(rows[2], W), 1 << 62]
    owner = [0, W - 1, 0, 1 % W]
    ol, oo, oi, op, _ = kernels.bucketize_rw(cu(ids), cu(offsets), F, B, W, cu(np.asarray(blocks, np.int64)),
                                             want_pos=True, feat_owner=cu(np.asarray(owner, np.int32)))
    wl, wo, wi, wp = O.bucketize_rw(ids, offsets, F, B, W, blocks, owner)
    np.testing.assert_array_equal(ol.cpu().numpy(), wl)
    np.testing.assert_array_equal(oi.cpu().numpy(), wi)
    np.testing.assert_array_equal(op.cpu().numpy(), wp)
    # every id of a table-wise feature landed on its owner, unchanged
    lens = wl.reshape(W, F, B)
    assert lens[:, 1].sum() == lens[owner[1], 1].sum() and lens[:, 3].sum() == lens[owner[3], 3].sum()


@pytest.mark.parametrize("pool", [O.POOL_SUM, O.POOL_MEAN])
def test_bag_grad_expand(kernels, pool):
    rng = np.random.default_rng(31)
    F, B, D = 5, 123, 16
    ids, lengths, offsets = random_kjt(rng, F, B, [100] * F, 4)
    lay = build_layout([100] * F, [D] * F, list(range(F)), [pool] * F).to(DEV)
    slot = rng.permutation(len(ids)).astype(np.int32)
    grad = rng.standard_normal((B, F * D)).astype(np.float32)
    got = kernels.bag_grad_expand(cu(grad), lay, cu(offsets), cu(slot), B, len(ids)).cpu().numpy()
    want = O.bag_grad_expand(grad, lay.col, lay.pool, offsets, slot, F, B, D, len(ids))
    np.testing.assert_array_equal(got, want)


def test_kjt_permute_bit_exact(kernels):
    rng = np.random.default_rng(4)
    F, B = 7, 100
    ids, lengths, offsets = random_kjt(rng, F, B, [1000] * F, 5)
    perm = [3, 0, 6, 6, 1]
    wi, wl = O.kjt_permute(ids, lengths, perm, B)
    pl = kernels.permute_lengths(cu(lengths), cu(np.asarray(perm, np.int32)), B)
    np.testing.assert_array_equal(pl.cpu().numpy(), wl)
    po = kernels.lengths_to_offsets(pl)
    pi = kernels.permute_ids(cu(ids), cu(offsets), po, cu(np.asarray(perm, np.int32)), B, len(wi))
    np.testing.assert_array_equal(pi.cpu().numpy(), wi)


def test_col_gather_sum_regroup_fwd_and_bwd(kernels):
    rng = np.random.default_rng(6)
    B = 77
    kt = rng.standard_normal((B, 104 + 416)).astype(np.float32)   # DeepFM: 26 wide(4) + 26 deep(16)
    dense = rng.standard_normal((B, 13)).astype(np.float32)
    # group "deep" = 13 dense cols then the 416 emb cols ; group "fm" = the 416 emb cols
    plan_deep = ColPlan(list(range(13 + 416 + 1)), [1] * 13 + [0] * 416, list(range(13)) + list(range(104, 520))).to(DEV)
    got = kernels.col_gather_sum([cu(kt), cu(dense)], plan_deep, B).cpu().numpy()
    np.testing.assert_array_equal(got, np.concatenate([dense, kt[:, 104:]], axis=1))
    # backward into kt: wide cols <- g_wide ; emb cols <- g_fm + g_deep[:, 13:]
    g_wide = rng.standard_normal((B, 104)).astype(np.float32)
    g_fm = rng.standard_normal((B, 416)).astype(np.float32)
    g_deep = rng.standard_normal((B, 429)).astype(np.float32)
    start, src, scol = [0], [], []
    for c in range(520):
        if c < 104:
            src += [0]; scol += [c]
        else:
            src += [1, 2]; scol += [c - 104, 13 + c - 104]
        start.append(len(src))
    plan_bwd = ColPlan(start, src, scol).to(DEV)
    gk = kernels.col_gather_sum([cu(g_wide), cu(g_fm), cu(g_deep)], plan_bwd, B).cpu().numpy()
    want = np.concatenate([g_wide, g_fm + g_deep[:, 13:]], axis=1)
    np.testing.assert_array_equal(gk, want)


def test_jagged_padded_round_trip(kernels):
    rng = np.random.default_rng(8)
    B, D = 50, 16
    lengths = rng.integers(0, 101, size=B).astype(np.int32)
    lengths[:3] = [0, 100, 1]
    offsets = O.lengths_to_offsets(lengths)
    vals = rng.standard_normal((int(offsets[-1]), D)).astype(np.float32)
    for T in [int(lengths.max()), 10, 1]:
        got = kernels.jagged_to_padded(cu(vals), cu(offsets), T).cpu().numpy()
        np.testing.assert_array_equal(got, O.to_padded_dense(vals, offsets, T))
        g = rng.standard_normal((B, T, D)).astype(np.float32)
        back = kernels.padded_to_jagged(cu(g), cu(offsets), len(vals)).cpu().numpy()
        np.testing.assert_array_equal(back, O.padded_to_jagged(g, offsets, len(vals)))


@pytest.mark.parametrize("tag", ["fm_criteo", "fm_small", "fm_wide"])
def test_fm_matches_reference_golden(kernels, tag):
    x, y, dy, dx = (GOLD[f"{tag}_{k}"] for k in ("x", "y", "dy", "dx"))
    B, N, D = x.shape
    got = kernels.fm_fwd(cu(x.reshape(B, N * D)), N, D).cpu().numpy()
    np.testing.assert_allclose(got, y, rtol=1e-5, atol=1e-5)
    gdx = kernels.fm_bwd(cu(x.reshape(B, N * D)), cu(dy), N, D).cpu().numpy()
    np.testing.assert_allclose(gdx.reshape(B, N, D), dx, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("tag", ["ia_criteo", "ia_min", "ia_odd", "ia_wide"])
def test_dot_interaction_matches_reference_golden(kernels, tag):
    x, z, dz, dx = (GOLD[f"{tag}_{k}"] for k in ("x", "z", "dz", "dx"))
    B, N, D = x.shape
    xs = cu(x.reshape(B, N * D))
    got = kernels.dot_interact_fwd(None, xs, N, D, False, False).cpu().numpy()
    np.testing.assert_allclose(got, z, rtol=1e-5, atol=1e-5)
    _, ds = kernels.dot_interact_bwd(None, xs, cu(dz), N, D, False, False)
    np.testing.assert_allclose(ds.cpu().numpy().reshape(B, N, D), dx, rtol=1e-5, atol=2e-5)


def test_dlrm_fused_interaction_vs_reference_golden_and_oracle(kernels):
    sparse, all_feat = GOLD["dlrm_sparse"], GOLD["dlrm_all_feat"]
    dense_feat = all_feat[:, 351:367]
    got = kernels.dot_interact_fwd(cu(dense_feat), cu(sparse), 26, 16, True, True).cpu().numpy()
    np.testing.assert_allclose(got, all_feat, rtol=1e-5, atol=1e-5)
    rng = np.random.default_rng(1)
    d_out = rng.standard_normal(all_feat.shape).astype(np.float32)
    dd, ds = kernels.dot_interact_bwd(cu(dense_feat), cu(sparse), cu(d_out), 26, 16, True, True)
    wd, ws = O.dlrm_interact_bwd(dense_feat, sparse, d_out, 26, 16)
    np.testing.assert_allclose(dd.cpu().numpy(), wd, rtol=1e-5, atol=2e-5)
    np.testing.assert_allclose(ds.cpu().numpy(), ws, rtol=1e-5, atol=2e-5)


def test_fused_bwd_ignores_zero_row_padding_features(kernels, bwd_path):
    """Static-capacity exchange: ids of a zero-row feature are wire padding — sorted last, never applied."""
    from torcheasyrec_b200.kernels import FeatureLayout

    rng = np.random.default_rng(77)
    rows, D, B = [400, 0, 50, 0], 16, 1            # B=1 "bags" = whole (source, feature) runs, as on the owner side
    lens = np.array([300, 5000, 200, 4000], dtype=np.int32)
    offsets = O.lengths_to_offsets(lens)
    ids = np.concatenate([rng.integers(0, max(r, 1), size=n) for r, n in zip(rows, lens)]).astype(np.int64)
    tables = [O.default_table_init(max(r, 1), D, rng)[:r] for r in rows]
    real = build_layout([400, 50], [D, D], [0, 1], [0, 0])
    lay = FeatureLayout(w_off=[real.w_off[0], 0, real.w_off[1], 0], rows=rows, dim=[D] * 4, col=[0] * 4, pool=[0] * 4,
                        key_base=[real.key_base[0], 0, real.key_base[1], 0], total_keys=real.total_keys,
                        total_dim=D, arena_elems=real.arena_elems).to(DEV)
    arena_np = np.zeros(real.arena_elems, np.float32)
    arena_np[real.w_off[0]:real.w_off[0] + 400 * D] = tables[0].ravel()
    arena_np[real.w_off[1]:real.w_off[1] + 50 * D] = tables[2].ravel()
    arena = cu(arena_np)
    state = torch.zeros_like(arena)
    grad = rng.standard_normal((len(ids), D)).astype(np.float32)
    kernels.fused_bwd(O.OPT_ADAGRAD, False, cu(grad), arena, state, lay, cu(ids), cu(offsets), B, 0.05, 1e-8, 1.0)
    want = [t.copy() for t in tables]
    st = [np.zeros_like(t) for t in tables]
    O.fused_update(O.OPT_ADAGRAD, want, st, [0, 1, 2, 3], [0] * 4, ids, offsets, B, grad, 0.05, 1e-8, 1.0, pooled=False)
    got = arena.cpu().numpy()
    np.testing.assert_allclose(got[real.w_off[0]:real.w_off[0] + 400 * D].reshape(400, D), want[0], rtol=5e-5, atol=5e-6)
    np.testing.assert_allclose(got[real.w_off[1]:real.w_off[1] + 50 * D].reshape(50, D), want[2], rtol=5e-5, atol=5e-6)


@pytest.mark.parametrize("W,factor", [(2, 1.5), (8, 2.5), (8, 1.2)])
def test_bucketize_fixed_capacity_wire_layout(kernels, W, factor):
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from oracle_backend import OracleKernels

    rng = np.random.default_rng(W + 100)
    F, B = 4, 500
    rows = [100000, 3, 77, 40000]
    ids, lengths, offsets = random_kjt(rng, F, B, rows, 1, fixed_len=1)
    blocks = np.asarray([O.rw_block_size(r, W) for r in rows], np.int64)
    C = int(factor * len(ids) / W) // 8 * 8 + 8      # factor 1.2 overflows on purpose (tiny tables skew the ranks)
    ol, oo, oi, op, inv = kernels.bucketize_rw(cu(ids), cu(offsets), F, B, W, cu(blocks), want_pos=True, want_inv=True,
                                               wire_capacity=C)
    wl, wo, wi, wp, winv = OracleKernels().bucketize_rw(torch.from_numpy(ids), torch.from_numpy(offsets), F, B, W,
                                                        torch.from_numpy(blocks), want_pos=True, want_inv=True,
                                                        wire_capacity=C)
    np.testing.assert_array_equal(ol.cpu().numpy(), wl.numpy())
    np.testing.assert_array_equal(oi.cpu().numpy(), wi.numpy())
    np.testing.assert_array_equal(op.cpu().numpy(), wp.numpy())
    np.testing.assert_array_equal(inv.cpu().numpy(), winv.numpy())
    per_dest = np.diff(wo.numpy()[::F * B])
    if (per_dest <= C).all():      # no overflow: every id is recoverable from its padded slot
        dest = inv.cpu().numpy() // C
        f_of = np.repeat(np.arange(F), B)
        np.testing.assert_array_equal(oi.cpu().numpy()[inv.cpu().numpy()] + dest * blocks[f_of], ids)
    else:
        assert factor < 1.5


def test_dlrm_interaction_aligned_layout_matches_reference_layout(kernels):
    """[P | 1 zero | dense | sparse] (784 wide) carries exactly the reference's 783 columns; same for the backward."""
    sparse, all_feat = GOLD["dlrm_sparse"], GOLD["dlrm_all_feat"]
    dense_feat = all_feat[:, 351:367]
    got = kernels.dot_interact_fwd(cu(dense_feat), cu(sparse), 26, 16, True, True, pad_to=4, p_pad=1).cpu().numpy()
    assert got.shape == (all_feat.shape[0], 784)
    np.testing.assert_allclose(got[:, :351], all_feat[:, :351], rtol=1e-5, atol=1e-5)
    assert (got[:, 351] == 0).all()
    np.testing.assert_array_equal(got[:, 352:], all_feat[:, 351:])
    rng = np.random.default_rng(2)
    d_out = rng.standard_normal(all_feat.shape).astype(np.float32)
    d_pad = np.concatenate([d_out[:, :351], rng.standard_normal((d_out.shape[0], 1)).astype(np.float32), d_out[:, 351:]], 1)
    dd, ds = kernels.dot_interact_bwd(cu(dense_feat), cu(sparse), cu(d_pad), 26, 16, True, True, p_pad=1)
    wd, ws = O.dlrm_interact_bwd(dense_feat, sparse, d_out, 26, 16)
    np.testing.assert_allclose(dd.cpu().numpy(), wd, rtol=1e-5, atol=2e-5)
    np.testing.assert_allclose(ds.cpu().numpy(), ws, rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize("N", [1, 16, 64, 256])
def test_tower_helpers_bias_act_and_relu_bwd_colsum(kernels, N):
    torch.manual_seed(N)
    M = 5000
    y = torch.randn(M, N, device=DEV)
    b = torch.randn(N, device=DEV)
    want = torch.relu(y + b)
    got = kernels.bias_act(y.clone(), b, True)
    assert torch.equal(got, want)
    dy = torch.randn(M, N, device=DEV)
    dz, colsum = kernels.act_bwd_colsum(dy, want, True)
    assert torch.equal(dz, dy * (want > 0))
    ref = (dy * (want > 0)).double().sum(0)
    np.testing.assert_allclose(colsum.cpu().numpy(), ref.cpu().numpy(), rtol=1e-5, atol=1e-4)
    _, cs2 = kernels.act_bwd_colsum(dy, None, False, want_dz=False)
    np.testing.assert_allclose(cs2.cpu().numpy(), dy.double().sum(0).cpu().numpy(), rtol=1e-5, atol=1e-4)


@pytest.fixture(params=["rows", "tile", "rows+dw_tiles"])
def slb_path(request, monkeypatch):
    """Both backward implementations behind tzk_small_linear_bwd: the barrier-free dx / dW kernels (default where the
    shape is covered) and the 128-row shared-memory tile kernel (TZK_SMALL_LINEAR_BWD=1; also the fallback)."""
    monkeypatch.setenv("TZK_SMALL_LINEAR_BWD", "1" if request.param == "tile" else "2")
    monkeypatch.setenv("TZK_SMALL_LINEAR_DW", "1" if request.param == "rows+dw_tiles" else "0")
    return request.param


@pytest.mark.parametrize("M,K,N,relu", [(1, 13, 64, True), (127, 64, 16, True), (128, 64, 32, True),
                                        (129, 32, 1, False), (1000, 3, 5, True), (4099, 64, 64, True),
                                        (300, 17, 33, False), (2500, 40, 2, True), (65536 + 7, 64, 32, True)])
def test_small_linear_fwd_bwd_vs_fp64_reference(kernels, slb_path, M, K, N, relu):
    """tzk_small_linear_{fwd,bwd} (the narrow tower layers) against a float64 restatement of
    tzrec/modules/mlp.py Perceptron: Linear -> ReLU and its autograd."""
    rng = np.random.default_rng(M * 7 + K * 3 + N)
    wide = rng.standard_normal((M, K + 5)).astype(np.float32)     # x is a column slice of a wider buffer
    x = cu(wide)[:, 2:2 + K]
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    dy = rng.standard_normal((M, N)).astype(np.float32)
    x64, w64, b64, dy64 = wide[:, 2:2 + K].astype(np.float64), w.astype(np.float64), b.astype(np.float64), dy.astype(np.float64)
    z = x64 @ w64.T + b64
    y64 = np.maximum(z, 0) if relu else z
    got = kernels.small_linear_fwd(x, cu(w), cu(b), relu)
    np.testing.assert_allclose(got.cpu().numpy(), y64, rtol=1e-5, atol=1e-5)
    dx, dw, db = kernels.small_linear_bwd(x, cu(w), got if relu else None, cu(dy), relu, True, True)
    dz = dy64 * (got.cpu().numpy() > 0) if relu else dy64
    np.testing.assert_allclose(dx.cpu().numpy(), dz @ w64, rtol=1e-5, atol=1e-5)
    scale = np.sqrt(M)
    np.testing.assert_allclose(dw.cpu().numpy(), dz.T @ x64, rtol=2e-5, atol=2e-5 * scale)
    np.testing.assert_allclose(db.cpu().numpy(), dz.sum(0), rtol=2e-5, atol=2e-5 * scale)
    # no-bias / no-dx variant and run-to-run determinism of the partial reduction
    y2 = kernels.small_linear_fwd(x, cu(w), None, relu)
    np.testing.assert_allclose(y2.cpu().numpy(), np.maximum(x64 @ w64.T, 0) if relu else x64 @ w64.T, rtol=1e-5, atol=1e-5)
    dx2, dw2, db2 = kernels.small_linear_bwd(x, cu(w), got if relu else None, cu(dy), relu, False, False)
    assert dx2 is None and db2 is None
    assert torch.equal(dw2, dw)


@pytest.mark.parametrize("M", [1, 5, 1023, 1024, 1025, 65536 + 3])
def test_bce_logits_fwd_bwd_matches_torch(kernels, M):
    torch.manual_seed(M)
    z = (torch.randn(M, device=DEV) * 6).requires_grad_(True)
    z.data[:min(M, 3)] = torch.tensor([40.0, -40.0, 0.0], device=DEV)[:min(M, 3)]
    t = (torch.rand(M, device=DEV) < 0.3).float()
    ref = torch.nn.functional.binary_cross_entropy_with_logits(z.double(), t.double())
    (gref,) = torch.autograd.grad(ref, z)
    loss, dz = kernels.bce_logits_fwd_bwd(z.detach(), t)
    np.testing.assert_allclose(float(loss), float(ref), rtol=1e-6)
    np.testing.assert_allclose(dz.cpu().numpy(), gref.float().cpu().numpy(), rtol=1e-5, atol=1e-9)


def test_linear_dispatch_and_bce_autograd_match_torch():
    """dense_gemm.linear / bce_with_logits (what the model shells call) against torch autograd, fp32."""
    from torcheasyrec_b200 import dense_gemm as G

    torch.manual_seed(5)
    B = 777
    x = torch.randn(B, 13, device=DEV)
    l1, l2, l3 = torch.nn.Linear(13, 64).to(DEV), torch.nn.Linear(64, 16).to(DEV), torch.nn.Linear(16, 1).to(DEV)
    t = (torch.rand(B, device=DEV) < 0.4).float()

    def run(fused):
        for m in (l1, l2, l3):
            m.zero_grad()
        if fused:
            h = G.linear(G.linear(x, l1.weight, l1.bias, relu=True), l2.weight, l2.bias, relu=True)
            loss = G.bce_with_logits(G.linear(h, l3.weight, l3.bias).squeeze(1), t)
        else:
            h = torch.relu(l2(torch.relu(l1(x))))
            loss = torch.nn.functional.binary_cross_entropy_with_logits(l3(h).squeeze(1), t)
        loss.backward()
        return float(loss), [p.grad.clone() for m in (l1, l2, l3) for p in m.parameters()]

    la, ga = run(True)
    lb, gb = run(False)
    assert abs(la - lb) <= 1e-6 * max(1.0, abs(lb))
    for a, b in zip(ga, gb):
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize("opt", [O.OPT_ADAM, O.OPT_PARTIAL_ROWWISE_ADAM])
@pytest.mark.parametrize("case", ["deepfm_mixed_dims", "tiny_tables_long_runs", "wide_rows", "unaligned_dims"])
def test_fused_bwd_adam_variants(kernels, case, opt, bwd_path):
    """tzk_fused_bwd_ex: Adam / partial row-wise Adam with weight decay and gradient clipping, three steps (the
    device-side step counter drives the bias correction), against the oracle (pinned to torch.optim.SparseAdam)."""
    rows, dims, feat_table, B, max_len = CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()) % 1000 + opt)
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    F = len(feat_table)
    frows = [rows[t] for t in feat_table]
    lay = build_layout(rows, dims, feat_table, [O.POOL_SUM] * F).to(DEV)
    arena = cu(make_arena(lay, tables, feat_table))
    m1 = torch.zeros_like(arena)
    m2 = torch.zeros_like(arena) if opt == O.OPT_ADAM else torch.zeros(lay.total_keys, device=DEV)
    step = torch.zeros((), device=DEV)
    want = [t.copy() for t in tables]
    s1 = [np.zeros_like(t) for t in tables]
    s2 = [np.zeros_like(t) if opt == O.OPT_ADAM else np.zeros(t.shape[0], np.float32) for t in tables]
    lr, eps, b1, b2, wd, mg = 0.02, 1e-8, 0.9, 0.999, 0.01, 0.7
    for it in range(1, 4):
        ids, lengths, offsets = random_kjt(rng, F, B, frows, max_len or 1, fixed_len=1 if max_len is None else None)
        grad = rng.standard_normal((B, lay.total_dim)).astype(np.float32)
        step.add_(1.0)
        kernels.fused_bwd(opt, True, cu(grad), arena, m1, lay, cu(ids), cu(offsets), B, lr, eps, 1.0, state2=m2,
                          step=step, beta1=b1, beta2=b2, weight_decay=wd, max_gradient=mg)
        O.fused_update(opt, want, s1, feat_table, [O.POOL_SUM] * F, ids, offsets, B, grad, lr, eps, 1.0, states2=s2,
                       step=it, beta1=b1, beta2=b2, weight_decay=wd, max_gradient=mg)
    got = split_arena(arena.cpu().numpy(), lay, tables, feat_table)
    for t in range(len(tables)):
        np.testing.assert_allclose(got[t], want[t], rtol=5e-5, atol=5e-6, err_msg=f"table {t}")
    gm = split_arena(m1.cpu().numpy(), lay, tables, feat_table)
    for t in range(len(tables)):
        np.testing.assert_allclose(gm[t], s1[t], rtol=5e-5, atol=1e-6)


def test_gradient_clipping_on_classic_optimizers(kernels, bwd_path):
    rng = np.random.default_rng(123)
    rows, dims, feat_table, B = [7, 300], [16, 16], [0, 1], 400
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    ids, lengths, offsets = random_kjt(rng, 2, B, rows, 3)
    lay = build_layout(rows, dims, feat_table, [0, 0]).to(DEV)
    arena = cu(make_arena(lay, tables, feat_table))
    state = torch.zeros_like(arena)
    grad = rng.standard_normal((B, 32)).astype(np.float32)
    kernels.fused_bwd(O.OPT_ADAGRAD, True, cu(grad), arena, state, lay, cu(ids), cu(offsets), B, 0.1, 1e-8, 1.0,
                      max_gradient=0.5)
    want, st = [t.copy() for t in tables], [np.zeros_like(t) for t in tables]
    O.fused_update(O.OPT_ADAGRAD, want, st, feat_table, [0, 0], ids, offsets, B, grad, 0.1, 1e-8, 1.0, max_gradient=0.5)
    got = split_arena(arena.cpu().numpy(), lay, tables, feat_table)
    for t in range(2):
        np.testing.assert_allclose(got[t], want[t], rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize("M", [300, 65536 + 5])
def test_gemm3x_kernels_match_fp64(monkeypatch, M):
    """csrc/tzk_gemm3x.cu (libtzk_gemm3x.so), the three passes of the 783 -> 64 tower layer on hand-written TMA-fed
    mma.sync TF32 kernels with the 3xTF32 split: forward (bias + ReLU epilogue), dgrad (W^T), wgrad (dZ^T X straight
    from the row-major tensors, bit-repeatable slab reduction).  fp32-level error against float64 — the same bound torch's fp32 SIMT GEMM meets."""
    from torcheasyrec_b200 import dense_gemm as G

    lib = G._gemm3x_lib()
    if lib is None:
        pytest.fail("libtzk_gemm3x.so missing: build() did not produce it")
    torch.manual_seed(M)
    K, N = 784, 64
    x = torch.randn(M, K, device=DEV)
    w = torch.randn(N, K, device=DEV) / K ** 0.5
    b = torch.randn(N, device=DEV)
    y = G.gemm3x(lib, x, w, b, True)
    ref = torch.relu(x.double() @ w.double().T + b.double())
    np.testing.assert_allclose(y.cpu().numpy(), ref.cpu().numpy(), atol=1.5e-5)
    dz = torch.randn(M, N, device=DEV)
    dx = G.gemm3x(lib, dz, w.t().contiguous(), None, False)
    np.testing.assert_allclose(dx.cpu().numpy(), (dz.double() @ w.double()).cpu().numpy(), atol=1.5e-5)
    dzs = dz / max(M, 1) ** 0.5
    dw = G.wgrad3x(lib, x, dzs)
    np.testing.assert_allclose(dw.cpu().numpy(), (dzs.double().T @ x.double()).cpu().numpy(), atol=1.5e-5)
    assert torch.equal(dw, G.wgrad3x(lib, x, dzs))


@pytest.mark.skipif(os.environ.get("TZK_TEST_GEMM3X_GLUE", "1") != "1",
                    reason="autograd glue of TZK_GEMM3X=1 (dense_gemm.Gemm3xLinearFn): covered on the CPU through the "
                           "emulated kernels; its first run on hardware is opted into with TZK_TEST_GEMM3X_GLUE=1")
@pytest.mark.parametrize("M", [300, 65536 + 5])
def test_wide_layer_on_tcgen05_matches_fp64(monkeypatch, M):
    """TZK_GEMM3X=1: the 783 -> 64 tower layer (input travelling as [B, 784] with a zero column) through
    dense_gemm.linear — forward with fused bias + ReLU, dgrad, wgrad — against float64 autograd.  (The name is that of
    the layer's first, Blackwell implementation; the test is the same for the Hopper kernels.)"""
    from torcheasyrec_b200 import dense_gemm as G

    if G._gemm3x_lib() is None:
        pytest.fail("libtzk_gemm3x.so missing: build() did not produce it")
    monkeypatch.setenv("TZK_GEMM3X", "1")
    torch.manual_seed(M)
    K, Kx, N = 783, 784, 64
    in_map = ((0, 0, 16), (16, 17, 767))
    xs = torch.randn(M, K, device=DEV)
    x = torch.zeros(M, Kx, device=DEV)
    for src, dst, n in in_map:
        x[:, dst:dst + n] = xs[:, src:src + n]
    x.requires_grad_(True)
    lin = torch.nn.Linear(K, N).to(DEV)
    y = G.linear(x, lin.weight, lin.bias, relu=True, in_map=in_map)
    g = torch.randn(M, N, device=DEV)
    y.backward(g)
    xr = xs.double().requires_grad_(True)
    wr, br = lin.weight.detach().double().requires_grad_(True), lin.bias.detach().double().requires_grad_(True)
    ref = torch.relu(torch.nn.functional.linear(xr, wr, br))
    ref.backward(g.double())
    np.testing.assert_allclose(y.detach().cpu().numpy(), ref.detach().cpu().numpy(), atol=2e-5)
    dx = torch.cat([x.grad[:, dst:dst + n] for _, dst, n in in_map], dim=1)
    np.testing.assert_allclose(dx.cpu().numpy(), xr.grad.cpu().numpy(), atol=2e-5)
    scale = float(M) ** 0.5
    np.testing.assert_allclose(lin.weight.grad.cpu().numpy(), wr.grad.cpu().numpy(), atol=2e-5 * scale)
    np.testing.assert_allclose(lin.bias.grad.cpu().numpy(), br.grad.cpu().numpy(), atol=2e-5 * scale)


@pytest.mark.parametrize("B,Ds,Dq,max_len,max_rows", [(1, 16, 16, 0, 5), (37, 48, 48, 0, 100), (300, 24, 8, 4, 9),
                                                      (8192, 48, 48, 0, 100), (64, 33, 33, 0, 40)])
def test_din_jagged_kernels_match_oracle(kernels, B, Ds, Dq, max_len, max_rows):
    """csrc/tzk_din.cu (SURVEY §8f N3) against the numpy restatement that the reference-generated DIN vectors pin
    (tests/test_model_blocks_pinning.py::test_jagged_din_attention_matches_the_reference_module): ragged lengths incl.
    empty samples, query narrower than the rows, max_seq_length truncation."""
    rng = np.random.default_rng(B * 7 + Ds)
    lens = rng.integers(0, max_rows + 1, B)
    lens[rng.integers(0, B)] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    N = int(off[-1])
    q = rng.standard_normal((B, Dq)).astype(np.float32)
    k = rng.standard_normal((N, Ds)).astype(np.float32)
    d_in = rng.standard_normal((N, 4 * Ds)).astype(np.float32)
    sc = (rng.standard_normal(N) * 3).astype(np.float32)
    d_out = rng.standard_normal((B, Ds)).astype(np.float32)
    from oracle_backend import OracleKernels

    ok = OracleKernels()
    tq, tk, toff = torch.from_numpy(q), torch.from_numpy(k), torch.from_numpy(off)
    want_in = ok.din_attn_input_fwd(tq, tk, toff)
    got_in = kernels.din_attn_input_fwd(cu(q), cu(k), cu(off))
    assert torch.equal(got_in.cpu(), want_in)
    wdq, wdk = ok.din_attn_input_bwd(torch.from_numpy(d_in), tq, tk, toff)
    gdq, gdk = kernels.din_attn_input_bwd(cu(d_in), cu(q), cu(k), cu(off))
    np.testing.assert_allclose(gdk.cpu().numpy(), wdk.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(gdq.cpu().numpy(), wdq.numpy(), rtol=2e-5, atol=2e-5)
    wp, wo = ok.jagged_softmax_wsum_fwd(torch.from_numpy(sc), tk, toff, max_len)
    gp, go = kernels.jagged_softmax_wsum_fwd(cu(sc), cu(k), cu(off), max_len)
    np.testing.assert_allclose(gp.cpu().numpy(), wp.numpy(), rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(go.cpu().numpy(), wo.numpy(), rtol=2e-5, atol=2e-6)
    wds, wdk2 = ok.jagged_softmax_wsum_bwd(torch.from_numpy(d_out), wp, tk, toff, max_len)
    gds, gdk2 = kernels.jagged_softmax_wsum_bwd(cu(d_out), gp, cu(k), cu(off), max_len)
    np.testing.assert_allclose(gds.cpu().numpy(), wds.numpy(), rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(gdk2.cpu().numpy(), wdk2.numpy(), rtol=2e-5, atol=1e-7)
    # run-to-run deterministic
    gp2, go2 = kernels.jagged_softmax_wsum_fwd(cu(sc), cu(k), cu(off), max_len)
    assert torch.equal(go, go2) and torch.equal(gp, gp2)


@pytest.mark.parametrize("opt", [O.OPT_SGD, O.OPT_ADAGRAD, O.OPT_ROWWISE_ADAGRAD, O.OPT_ADAM])
def test_fp16_tables_gather_and_fused_update(kernels, opt):
    """SURVEY §8f N4 (FP16 half): an arena of halfs against the oracle run on the same halfs — lookups bit-exact at L=1
    and 1e-6 for multi-hot bags (fp32 pooling), sequence rows exact, the fused update in fp32 with the new row rounded
    to nearest half (weights compared at half precision, fp32 state at 1e-5)."""
    from oracle_backend import OracleKernels

    from torcheasyrec_b200.embedding_modules import (DataType, EmbeddingBagCollection, EmbeddingBagConfig,
                                                     SparseOptimizerSpec)

    rng = np.random.default_rng(opt)
    cfgs = [EmbeddingBagConfig(num_embeddings=r, embedding_dim=d, name=f"t{i}", feature_names=[f"f{i}"],
                               data_type=DataType.FP16) for i, (r, d) in enumerate([(5000, 16), (7, 16), (300, 4), (64, 16)])]
    gpu = EmbeddingBagCollection(cfgs, device="cuda")
    cpu = EmbeddingBagCollection(cfgs, device="cpu")
    assert gpu.weights.dtype == torch.float16 and gpu.table_weight(0).dtype == torch.float16
    cpu.weights.data.copy_(gpu.weights.data.cpu())
    kind = {O.OPT_SGD: "sgd", O.OPT_ADAGRAD: "adagrad", O.OPT_ROWWISE_ADAGRAD: "rowwise_adagrad", O.OPT_ADAM: "adam"}[opt]
    spec = SparseOptimizerSpec.from_name(kind, lr=0.05)
    gpu.set_optimizer(spec)
    cpu.set_optimizer(spec)
    F, B = 4, 700
    lens = rng.integers(0, 4, F * B)
    lens[:B] = 1
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rows = [c.num_embeddings for c in cfgs]
    ids = np.concatenate([rng.integers(0, rows[b // B], lens[b]) for b in range(F * B)]).astype(np.int64)
    lay = gpu.layout
    ok = OracleKernels()
    want = ok.pooled_gather_fwd(cpu.weights.data, cpu.layout, torch.from_numpy(ids), torch.from_numpy(off), B)
    got = kernels.pooled_gather_fwd(gpu.weights.data, lay, cu(ids), cu(off), B)
    np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
    assert np.array_equal(got.cpu().numpy()[:, :16], want.numpy()[:, :16])         # feature 0: one id per bag -> exact
    grad = (rng.standard_normal((B, lay.total_dim)) * 0.1).astype(np.float32)
    for step in range(2):
        kernels.fused_bwd(spec.kind, True, cu(grad), gpu.weights.data, gpu.opt_state, lay, cu(ids), cu(off), B, spec.lr,
                          spec.eps, 1.0, **gpu.opt_extras())
        ok.fused_bwd(spec.kind, True, torch.from_numpy(grad), cpu.weights.data, cpu.opt_state, cpu.layout,
                     torch.from_numpy(ids), torch.from_numpy(off), B, spec.lr, spec.eps, 1.0, **cpu.opt_extras())
    gw, cw = gpu.weights.data.float().cpu().numpy(), cpu.weights.data.float().numpy()
    # one half ulp is 2^-11 relative: a summation-order difference may flip the final rounding of a few elements
    np.testing.assert_allclose(gw, cw, rtol=1.5e-3, atol=1e-6)
    assert (gw != cw).mean() < 0.01
    if gpu.opt_state is not None:
        np.testing.assert_allclose(gpu.opt_state.cpu().numpy(), cpu.opt_state.numpy(), rtol=1e-4, atol=1e-7)


def test_fp16_sequence_collection_rows(kernels):
    from torcheasyrec_b200.embedding_modules import DataType, EmbeddingCollection, EmbeddingConfig

    rng = np.random.default_rng(1)
    cfgs = [EmbeddingConfig(num_embeddings=900, embedding_dim=16, name="s", feature_names=["a"], data_type=DataType.FP16)]
    ec = EmbeddingCollection(cfgs, device="cuda")
    B = 50
    lens = rng.integers(0, 9, B)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = rng.integers(0, 900, int(off[-1])).astype(np.int64)
    rows = kernels.seq_gather_fwd(ec.weights.data, ec.layout, cu(ids), cu(off), B)
    assert rows.dtype == torch.float32
    assert torch.equal(rows, ec.table_weight(0)[cu(ids)].float())


# Paths that have not been through a GPU validation pass yet run only when asked for (TZK_EXPERIMENTAL=1); a
# validated path loses the mark and gets its default flipped in the library.
unvalidated = pytest.mark.skipif(os.environ.get("TZK_EXPERIMENTAL") != "1",
                                 reason="unvalidated path: set TZK_EXPERIMENTAL=1")


# ---- interleaved [weight row | Adagrad accumulator row] arenas (tzk_opt_args.interleaved) -----------------------------------
def _interleaved_arena(lay, tables, states, feat_table):
    arena = np.zeros(lay.arena_elems, dtype=np.float32)
    for f, t in enumerate(feat_table):
        r, d = tables[t].shape
        v = arena[lay.w_off[f]:lay.w_off[f] + r * 2 * d].reshape(r, 2 * d)
        v[:, :d], v[:, d:] = tables[t], states[t]
    return arena


def _split_interleaved(arena, lay, tables, feat_table):
    w, s = {}, {}
    for f, t in enumerate(feat_table):
        r, d = tables[t].shape
        v = arena[lay.w_off[f]:lay.w_off[f] + r * 2 * d].reshape(r, 2 * d)
        w[t], s[t] = v[:, :d], v[:, d:]
    return [w[t] for t in range(len(tables))], [s[t] for t in range(len(tables))]


@pytest.mark.parametrize("case", ["criteo_like_L1", "deepfm_mixed_dims", "shared_table", "wide_rows", "unaligned_dims",
                                  "tiny_tables_long_runs", "multi_hot_33", "long_runs_d4"])
@pytest.mark.parametrize("pool", [O.POOL_SUM, O.POOL_MEAN])
def test_interleaved_gather_and_adagrad_update(kernels, case, pool):
    """The strided gather and the fused Adagrad update over [weight | state] lines against the oracle on dense tables:
    lookups bit-exact at L = 1, two update steps, weights AND accumulators compared, run-to-run identical bits."""
    rows, dims, feat_table, B, max_len = CASES[case]
    rng = np.random.default_rng(zlib.crc32(case.encode()) % 1000 + 91)
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    st_np = [np.abs(rng.standard_normal(t.shape)).astype(np.float32) * 0.01 for t in tables]
    F = len(feat_table)
    frows = [rows[t] for t in feat_table]
    ids, lengths, offsets = random_kjt(rng, F, B, frows, max_len or 1, fixed_len=1 if max_len is None else None)
    lay = build_layout(rows, dims, feat_table, [pool] * F, interleaved=True).to(DEV)
    assert lay.interleaved and all(lay.stride[f] == 2 * lay.dim[f] for f in range(F))
    arena0 = _interleaved_arena(lay, tables, st_np, feat_table)
    arena = cu(arena0)
    got = kernels.pooled_gather_fwd(arena, lay, cu(ids), cu(offsets), B).cpu().numpy()
    want_out = O.pooled_lookup(tables, feat_table, [pool] * F, ids, offsets, B)
    if pool == O.POOL_SUM and max_len is None:
        np.testing.assert_array_equal(got, want_out)
    np.testing.assert_allclose(got, want_out, rtol=1e-5, atol=1e-7)
    grad = rng.standard_normal((B, lay.total_dim)).astype(np.float32)
    lr, eps, gs = 0.05, 1e-8, 0.5
    long_runs = case in ("tiny_tables_long_runs", "long_runs_d4")
    state_rtol = 3e-4 if long_runs else 2e-5
    w_rtol, w_atol = (5e-5, 5e-6) if long_runs else (1e-5, 1e-6)
    want = [t.copy() for t in tables]
    twin = cu(arena0)
    for _ in range(2):
        kernels.fused_bwd(O.OPT_ADAGRAD, True, cu(grad), arena, None, lay, cu(ids), cu(offsets), B, lr, eps, gs)
        kernels.fused_bwd(O.OPT_ADAGRAD, True, cu(grad), twin, None, lay, cu(ids), cu(offsets), B, lr, eps, gs)
        O.fused_update(O.OPT_ADAGRAD, want, st_np, feat_table, [pool] * F, ids, offsets, B, grad, lr, eps, gs)
    assert torch.equal(arena, twin)
    gw, gs_ = _split_interleaved(arena.cpu().numpy(), lay, tables, feat_table)
    for t in range(len(tables)):
        np.testing.assert_allclose(gw[t], want[t], rtol=w_rtol, atol=w_atol, err_msg=f"table {t}")
        np.testing.assert_allclose(gs_[t], st_np[t], rtol=state_rtol, atol=1e-7, err_msg=f"state {t}")


def test_interleaved_split_sort_apply_and_sequence_layout(kernels):
    """The two halves of the fused backward (sort on the ids, apply on the gradient) and the un-pooled lookup / update."""
    rng = np.random.default_rng(77)
    rows, dims, feat_table, B = [400, 30, 400], [16, 16, 16], [0, 1, 2], 64
    tables = [O.default_table_init(r, d, rng) for r, d in zip(rows, dims)]
    st_np = [np.zeros_like(t) for t in tables]
    ids, lengths, offsets = random_kjt(rng, 3, B, rows, 12)
    lay = build_layout(rows, dims, feat_table, [0] * 3, interleaved=True).to(DEV)
    arena = cu(_interleaved_arena(lay, tables, st_np, feat_table))
    rows_out = kernels.seq_gather_fwd(arena, lay, cu(ids), cu(offsets), B).cpu().numpy()
    np.testing.assert_array_equal(rows_out, O.seq_lookup(tables, feat_table, ids, offsets, B))
    grad = rng.standard_normal((len(ids), 16)).astype(np.float32)
    ws = torch.empty(kernels.fused_bwd_workspace_bytes(lay, len(ids)), dtype=torch.uint8, device=DEV)
    kernels.fused_bwd_sort(False, lay, cu(ids), cu(offsets), B, ws)
    kernels.fused_bwd_apply(O.OPT_ADAGRAD, False, cu(grad), arena, None, lay, cu(offsets), len(ids), B, 0.02, 1e-8, 1.0, ws)
    want = [t.copy() for t in tables]
    O.fused_update(O.OPT_ADAGRAD, want, st_np, feat_table, [0] * 3, ids, offsets, B, grad, 0.02, 1e-8, 1.0, pooled=False)
    gw, gs_ = _split_interleaved(arena.cpu().numpy(), lay, tables, feat_table)
    for t in range(3):
        np.testing.assert_allclose(gw[t], want[t], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(gs_[t], st_np[t], rtol=2e-5, atol=1e-7)


def test_interleaved_rejects_what_it_does_not_cover(kernels):
    lay = build_layout([10], [16], [0], [0], interleaved=True).to(DEV)
    arena = torch.zeros(lay.arena_elems, device=DEV)
    ids, off = torch.zeros(4, dtype=torch.int64, device=DEV), torch.arange(5, dtype=torch.int64, device=DEV)
    grad = torch.zeros(4, 16, device=DEV)
    with pytest.raises(Exception, match="interleaved"):
        kernels.fused_bwd(O.OPT_ROWWISE_ADAGRAD, True, grad, arena, None, lay, ids, off, 4, 0.1, 1e-8, 1.0)


# ---- DLRM interaction on the tensor cores (csrc/tzk_interact_tc.cuh; TZK_INTERACT_TC=1) ------------------------------------
@pytest.mark.parametrize("B", [1, 8, 777, 40000])
def test_interaction_tensor_core_kernels_match_reference_and_fp64(kernels, monkeypatch, B):
    """mma.sync m16n8k8 with the 3xTF32 split, DLRM-Criteo shape (27 x 16, [351 | 0 | 16 | 416] rows): the reference's own
    golden vectors (B = the fixture's batch), float64 at other batch sizes, and the FFMA kernels of tzk_dense.cu."""
    sparse_g, all_feat = GOLD["dlrm_sparse"], GOLD["dlrm_all_feat"]
    rng = np.random.default_rng(B)
    if B == 8 and sparse_g.shape[0] >= 8:
        sparse, dense = sparse_g[:8], all_feat[:8, 351:367]
        want_fwd = all_feat[:8]
    else:
        sparse = rng.standard_normal((B, 416)).astype(np.float32)
        dense = rng.standard_normal((B, 16)).astype(np.float32)
        want_fwd = None
    d_pad = rng.standard_normal((B, 784)).astype(np.float32)
    monkeypatch.setenv("TZK_INTERACT_TC", "0")
    ref = kernels.dot_interact_fwd(cu(dense), cu(sparse), 26, 16, True, True, pad_to=4, p_pad=1)
    rdd, rds = kernels.dot_interact_bwd(cu(dense), cu(sparse), cu(d_pad), 26, 16, True, True, p_pad=1)
    monkeypatch.setenv("TZK_INTERACT_TC", "1")
    monkeypatch.setenv("TZK_INTERACT_TC_BWD", "1")
    got = kernels.dot_interact_fwd(cu(dense), cu(sparse), 26, 16, True, True, pad_to=4, p_pad=1)
    dd, ds = kernels.dot_interact_bwd(cu(dense), cu(sparse), cu(d_pad), 26, 16, True, True, p_pad=1)
    torch.cuda.synchronize()
    assert got.shape == (B, 784)
    assert torch.equal(got[:, 351:], ref[:, 351:])                     # zero + copy part: same bits
    x = np.concatenate([dense[:, None, :], sparse.reshape(B, 26, 16)], 1).astype(np.float64)
    z = x @ x.transpose(0, 2, 1)
    iu = np.triu_indices(27, 1)
    np.testing.assert_allclose(got[:, :351].cpu().numpy(), z[:, iu[0], iu[1]], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(got[:, :351], ref[:, :351], rtol=1e-5, atol=1e-5)
    if want_fwd is not None:
        np.testing.assert_allclose(got[:, :351].cpu().numpy(), want_fwd[:, :351], rtol=1e-5, atol=1e-5)
    G = np.zeros((B, 27, 27))
    G[:, iu[0], iu[1]] = d_pad[:, :351]
    dx = (G + G.transpose(0, 2, 1)) @ x + d_pad[:, 352:].astype(np.float64).reshape(B, 27, 16)
    np.testing.assert_allclose(dd.cpu().numpy(), dx[:, 0], rtol=1e-5, atol=3e-5)
    np.testing.assert_allclose(ds.cpu().numpy(), dx[:, 1:].reshape(B, -1), rtol=1e-5, atol=3e-5)
    torch.testing.assert_close(dd, rdd, rtol=1e-5, atol=3e-5)
    torch.testing.assert_close(ds, rds, rtol=1e-5, atol=3e-5)
    # run-to-run identical bits
    again = kernels.dot_interact_fwd(cu(dense), cu(sparse), 26, 16, True, True, pad_to=4, p_pad=1)
    assert torch.equal(again, got)


# ---- fused tower tail: last Perceptron + Linear(N, 1) + mean BCE, forward and backward in one kernel ---------------------
@pytest.mark.parametrize("M,K,N", [(1, 64, 32), (127, 64, 32), (1000, 13, 7), (4099, 64, 64), (65536 + 5, 64, 32), (300, 32, 16)])
def test_tower_tail_bce_matches_torch_autograd(kernels, M, K, N):
    """tzk_tower_tail_bce against torch autograd in float64 (tzrec/modules/mlp.py Perceptron -> Linear ->
    BCEWithLogitsLoss(mean)): loss, logits and every gradient; y1 as a column slice of a wider buffer."""
    from torcheasyrec_b200.dense_gemm import tower_tail_bce

    g = torch.Generator(device="cpu").manual_seed(M + K + N)
    wide = torch.relu(torch.randn(M, K + 4, generator=g)).to(DEV)
    y1 = wide[:, :K].detach().requires_grad_()
    w1 = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV).requires_grad_()
    b1 = (0.1 * torch.randn(N, generator=g)).to(DEV).requires_grad_()
    w2 = (torch.randn(1, N, generator=g) / N ** 0.5).to(DEV).requires_grad_()
    b2 = torch.tensor([0.05]).to(DEV).requires_grad_()
    lab = (torch.rand(M, generator=g) < 0.3).float().to(DEV)
    loss, logits = tower_tail_bce(y1, w1, b1, w2, b2, lab)
    (loss * 1.0).backward()
    ref_in = [t.detach().double().requires_grad_() for t in (y1, w1, b1, w2, b2)]
    h = torch.relu(ref_in[0] @ ref_in[1].t() + ref_in[2])
    z = (h @ ref_in[3].t() + ref_in[4]).squeeze(1)
    ref = torch.nn.functional.binary_cross_entropy_with_logits(z, lab.double())
    ref.backward()
    torch.testing.assert_close(loss.double(), ref, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(logits.double(), z.detach(), rtol=1e-5, atol=1e-5)
    for got, want, name in zip((y1, w1, b1, w2, b2), ref_in, ("dy1", "dW1", "db1", "dw2", "db2")):
        torch.testing.assert_close(got.grad.double(), want.grad, rtol=2e-4, atol=2e-7, msg=lambda m, n=name: f"{n}: {m}")
    # run-to-run identical bits
    y1b = wide[:, :K].detach().requires_grad_()
    loss2, _ = tower_tail_bce(y1b, w1.detach().requires_grad_(), b1, w2, b2, lab)
    assert torch.equal(loss2, loss)
