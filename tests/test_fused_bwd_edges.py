"""tzk_fused_bwd (csrc/tzk_bwd.cu) at its dispatch and run-length edges, against an exact float64 reference.

The kernel is a tree of paths picked on the host: key width (uint32 / uint64), VEC (4 or 1, from vec_ok and the actual
pointer alignment), lane group G and chunks per lane CH (from max_dim), the general path or the tile path
(TZK_BWD_TILE=1), the short-run head list or the walk over every position (TZK_BWD_HEADS=0), short / single-chunk /
multi-chunk runs, and the opt-in shared memory above 1228 features.  These tests place runs exactly and make every
row sum exact, so one dropped or doubled contribution changes the result's bits.

Exactness: gradient values are k * 2^-6 with small nonzero integer k, grad_scale is a power of two and MEAN bags have
lengths in {1, 2, 4, 8}, so every contribution g * scale is an exact multiple of the quantum q = grad_scale * 2^-9.
When the absolute contributions of a row add up to less than 2^24 q, every partial sum in any order is a multiple of q
below 2^24 q, hence exact in fp32: the fp32 sum equals the float64 sum bit for bit.  `check_exact` asserts this on the
constructed data.

Readout: SGD with lr = -1 on a zero arena stores w = 0 - (-1) * acc = acc, so after one call every touched row equals
its float64 row sum bit for bit and every untouched row is still 0.
"""
import zlib
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from torcheasyrec_b200._lib import TzkError
from torcheasyrec_b200.kernels import (OPT_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM, OPT_ROWWISE_ADAGRAD, OPT_SGD,
                                       POOL_MEAN, POOL_SUM, FeatureLayout)

DEV = "cuda"
Q = 2.0 ** -6                 # gradient grid
MEAN_LENS = (1, 2, 4, 8)      # bag lengths: g / L stays on the grid q = 2^-9
U = 2.0 ** -24                # fp32 unit roundoff
KEY32 = 1 << 32


# ---------------------------------------------------------------------------------------------------------------------
# host mirror of the dispatch in fused_bwd_impl (names the path each case takes)
def dispatch(max_dim, vec):
    """(G, CH) of the general path: G lanes per row, CH = compiled chunks per lane (1, 2 or 8); ch > 8 is rejected."""
    need = -(-max_dim // vec)
    g = 1
    while g < need and g < 32:
        g *= 2
    ch = -(-need // g)
    return g, (1 if ch == 1 else 2 if ch <= 2 else 8 if ch <= 8 else ch)


def tile_positions(g):
    """TP of TileCfg<G>: sorted positions per tile."""
    return 4096 // (4 * g)


# ---------------------------------------------------------------------------------------------------------------------
# layouts
def make_layout(tables, feat_table, pool, n_pad=0, key_bases=None, stored=None):
    """tables: [(rows, dim)]; features read feat_table[f]; `n_pad` zero-row "wire padding" features are appended (their
    ids sort to the sentinel tail).  key_bases: per-table key base (default: packed).  stored: rows per table that exist
    in the arena (a table may be declared with 2^32 rows and store only the few rows the test touches)."""
    stored = stored or [r for r, _ in tables]
    t_off, o = [], 0
    for (_, d), s in zip(tables, stored):
        o = (o + 3) // 4 * 4
        t_off.append(o)
        o += s * d
    if key_bases is None:
        key_bases, k = [], 0
        for r, _ in tables:
            key_bases.append(k)
            k += r
    total_keys = max(kb + r for kb, (r, _) in zip(key_bases, tables))
    w_off, rows, dim, col, pl, kb = [], [], [], [], [], []
    c = 0
    for t in feat_table:
        w_off.append(t_off[t]); rows.append(tables[t][0]); dim.append(tables[t][1]); col.append(c); pl.append(pool)
        kb.append(key_bases[t])
        c += tables[t][1]
    for _ in range(n_pad):
        d = tables[0][1]
        w_off.append(0); rows.append(0); dim.append(d); col.append(c); pl.append(pool); kb.append(0)
        c += d
    return FeatureLayout(w_off=w_off, rows=rows, dim=dim, col=col, pool=pl, key_base=kb, total_keys=total_keys,
                         total_dim=c, arena_elems=max(o, 128))


# ---------------------------------------------------------------------------------------------------------------------
# run placement: counts per key whose stable sort has the requested runs at the requested positions
def next_start(pos, where):
    """Smallest position >= pos that satisfies `where` = (modulus, residue) (None: any)."""
    if where is None:
        return pos
    m, r = where
    return pos + (r - pos) % m


def plan_runs(rng, specs, key0=0, pos0=0, filler=(1, 4), p_untouched=0.3):
    """specs: [(length, where)] in key order.  The run of spec i gets its own key; the gap before it is filled with
    short filler runs on the keys in between (some keys are left untouched).  Returns (keys, counts, placed) with
    placed[i] = (key, start position, length); positions count from pos0 (the hits of all lower keys)."""
    keys, counts, placed = [], [], []
    key, pos = key0, pos0
    for length, where in specs:
        start = next_start(pos, where)
        gap = start - pos
        while gap > 0:
            if rng.random() < p_untouched:
                key += 1                                   # an untouched row between runs
            n = int(min(gap, rng.integers(filler[0], filler[1] + 1)))
            keys.append(key); counts.append(n)
            key += 1
            gap -= n
        keys.append(key); counts.append(length)
        placed.append((key, start, length))
        key += 1
        pos = start + length
    return np.array(keys, np.int64), np.array(counts, np.int64), placed


def bag_lengths(rng, n):
    """Lengths in {1, 2, 4, 8} that add up to n."""
    if n == 0:
        return np.zeros(0, np.int64)
    lens = rng.choice(MEAN_LENS, size=n)
    cs = np.cumsum(lens)
    cut = int(np.searchsorted(cs, n))          # first index with cs >= n
    lens = lens[:cut + 1].copy()
    rest = n - (int(cs[cut - 1]) if cut else 0)
    lens = lens[:-1]
    tail = [b for b in (8, 4, 2, 1) if rest & b]
    return np.concatenate([lens, np.array(tail, np.int64)])


@dataclass
class Kjt:
    ids: np.ndarray
    offsets: np.ndarray
    B: int
    pooled: bool


def build_kjt(rng, lay, keys, counts, B_min=1, pooled=True, pad_ids=0):
    """ids / offsets (feature-major, F * B bags) in which key keys[i] is hit counts[i] times.  Each hit goes to a
    random feature that reads the key's table and to a random bag of it, so a run gathers contributions from many bags
    and features.  Pooled bags have lengths in {1, 2, 4, 8}; the zero-row padding features get `pad_ids` ids each."""
    F = lay.num_features
    real = [f for f in range(F) if lay.rows[f] > 0]
    hits = np.repeat(keys, counts)
    owner = np.full(len(hits), -1, np.int64)
    tabs = sorted({(lay.key_base[f], lay.rows[f]) for f in real})
    for kb, r in tabs:
        fs = [f for f in real if lay.key_base[f] == kb and lay.rows[f] == r]
        sel = (hits >= kb) & (hits < kb + r)
        owner[sel] = np.asarray(fs)[rng.integers(0, len(fs), int(sel.sum()))]
    assert (owner >= 0).all(), "a key outside every table"
    per_f = []
    for f in range(F):
        if lay.rows[f] > 0:
            ids_f = hits[owner == f] - lay.key_base[f]
            ids_f = ids_f[rng.permutation(len(ids_f))]
        else:
            ids_f = rng.integers(0, 7, pad_ids).astype(np.int64)
        per_f.append((ids_f, bag_lengths(rng, len(ids_f))))
    B = max([B_min] + [len(lens) for _, lens in per_f])
    lengths = np.zeros(F * B, np.int64)
    for f, (_, lens) in enumerate(per_f):
        slots = np.sort(rng.choice(B, size=len(lens), replace=False))
        lengths[f * B + slots] = lens[rng.permutation(len(lens))]
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    ids = np.concatenate([ids_f for ids_f, _ in per_f] + [np.zeros(0, np.int64)]).astype(np.int64)
    return Kjt(ids, offsets, B, pooled)


def grad_values(rng, shape, kmax=3):
    """k * 2^-6 with k in +-{1..kmax}: never zero, so a dropped contribution always shows."""
    k = rng.integers(1, kmax + 1, size=shape) * rng.choice([-1, 1], size=shape)
    return (k * Q).astype(np.float32)


def make_grad(rng, lay, kjt, kmax=3):
    rows = kjt.B if kjt.pooled else len(kjt.ids)
    return grad_values(rng, (rows, max(lay.total_dim if kjt.pooled else lay.max_dim, 1)), kmax)


# ---------------------------------------------------------------------------------------------------------------------
# the reference
def position_keys(lay, kjt):
    """Linearized key of every id position (the sort input); padding features get a key above every real one."""
    F, B = lay.num_features, kjt.B
    lens = np.diff(kjt.offsets)
    feat = np.repeat(np.arange(F * B) // B, lens)
    rows = np.asarray(lay.rows, np.int64)[feat]
    ids = np.where((kjt.ids >= 0) & (kjt.ids < rows), kjt.ids, 0)
    keys = np.asarray(lay.key_base, np.int64)[feat] + ids
    return np.where(rows > 0, keys, np.int64(2 ** 62)), feat


def contributions(lay, kjt, grad, gs):
    """Per real id position: its key and its gradient contribution g * scale (float64, [n, max_dim], zero beyond the
    feature's dim) exactly as the kernel forms it."""
    F, B = lay.num_features, kjt.B
    lens = np.diff(kjt.offsets)
    keys, feat = position_keys(lay, kjt)
    bag = np.repeat(np.arange(F * B), lens)
    real = np.asarray(lay.rows, np.int64)[feat] > 0
    n = len(kjt.ids)
    C = np.zeros((n, lay.max_dim), np.float64)
    for f in range(F):
        if lay.rows[f] == 0:
            continue
        s, e = int(kjt.offsets[f * B]), int(kjt.offsets[(f + 1) * B])
        if s == e:
            continue
        d = lay.dim[f]
        if kjt.pooled:
            g = grad[bag[s:e] - f * B, lay.col[f]:lay.col[f] + d].astype(np.float64)
            scale = gs / lens[bag[s:e]] if lay.pool[f] == POOL_MEAN else np.full(e - s, gs)
        else:
            g = grad[s:e, :d].astype(np.float64)
            scale = np.full(e - s, gs)
        C[s:e, :d] = g * scale[:, None]
    return keys[real], C[real]


def row_sums(lay, kjt, grad, gs, dtype=np.float64, order=None):
    """(unique keys, per-key sums [n_keys, max_dim]) summed in `dtype`, adding the positions in `order` (default:
    position order) one at a time."""
    keys, C = contributions(lay, kjt, grad, gs)
    uk, inv = np.unique(keys, return_inverse=True)
    S = np.zeros((len(uk), lay.max_dim), dtype)
    idx = np.arange(len(keys)) if order is None else order
    np.add.at(S, inv[idx], C[idx].astype(dtype))
    return uk, S


def check_exact(lay, kjt, grad, gs):
    """The exactness precondition, asserted from the data: every contribution is an integer multiple of
    q = gs * 2^-9 and, per row, the absolute contributions add up to less than 2^24 q."""
    m, e = np.frexp(gs)
    assert m == 0.5, f"grad_scale {gs} is not a power of two"
    assert set(np.unique(np.diff(kjt.offsets))) <= {0, *MEAN_LENS}
    q = gs * Q / 8
    keys, C = contributions(lay, kjt, grad, gs)
    units = C / q
    assert np.array_equal(units, np.round(units)), "a contribution is off the grid"
    uk, inv = np.unique(keys, return_inverse=True)
    A = np.zeros((len(uk), lay.max_dim))
    np.add.at(A, inv, np.abs(C))
    assert A.max(initial=0.0) < 2.0 ** 24 * q, "a row's partial sums could leave the exact fp32 range"
    return q


def expected_arena(lay, uk, S, base=None):
    """Arena after the readout: float32 row sums in the touched rows, `base` (default zeros) elsewhere."""
    out = np.zeros(lay.arena_elems, np.float32) if base is None else base.copy()
    for f in range(lay.num_features):
        if lay.rows[f] == 0:
            continue
        kb, d = lay.key_base[f], lay.dim[f]
        sel = (uk >= kb) & (uk < kb + lay.rows[f])
        for k, s in zip(uk[sel], S[sel]):
            o = lay.w_off[f] + (int(k) - kb) * d
            out[o:o + d] = s[:d]
    return out


def sorted_runs(lay, kjt, key):
    """(start, length) of `key`'s run in the stable sort of the position keys."""
    pk, _ = position_keys(lay, kjt)
    sk = pk[np.argsort(pk, kind="stable")]
    s = int(np.searchsorted(sk, key, "left"))
    return s, int(np.searchsorted(sk, key, "right")) - s


# ---------------------------------------------------------------------------------------------------------------------
# cases
RUN_LENGTHS = (1, 2, 31, 32, 33, 255, 256, 257, 512, 513)
WARP_STARTS = ((32, 0), (32, 1), (32, 31))


def tile_starts(tp):
    return ((tp, tp - 1), (tp, 0), (tp, 1))


def run_specs(g):
    """Every run length at every start class: warp (ballot) boundaries of the head list and tile boundaries of
    TileCfg<g>; plus runs of TP - 1, TP, TP + 1 and 2 TP + 1 positions (the last spans a whole middle tile)."""
    tp = tile_positions(g)
    lengths = RUN_LENGTHS + (tp - 1, tp, tp + 1, 2 * tp + 1)
    return [(n, w) for n in lengths for w in WARP_STARTS + tile_starts(tp)]


def edge_case(seed, dim, pooled, n_pad=0):
    """One table (dim `dim`) read by two features, runs from run_specs(G) at their start classes."""
    rng = np.random.default_rng(seed)
    g, _ = dispatch(dim, 4 if dim % 4 == 0 else 1)
    specs = run_specs(g)
    keys, counts, placed = plan_runs(rng, specs)
    lay = make_layout([(int(keys[-1]) + 3, dim)], [0, 0], POOL_MEAN if pooled else POOL_SUM, n_pad=n_pad)
    kjt = build_kjt(rng, lay, keys, counts, pooled=pooled, pad_ids=500)
    grad = make_grad(rng, lay, kjt)
    return lay, kjt, grad, placed


def sweep_case(seed, dims, pooled=True):
    """One table per dim, two features each; runs of 1, 3, 32, 33, 257 and 300 positions next to random short runs."""
    rng = np.random.default_rng(seed)
    tables = [(48, d) for d in dims]
    feat_table = [t for t in range(len(dims)) for _ in range(2)]
    lay = make_layout(tables, feat_table, POOL_MEAN)
    ks, cs = [], []
    for t in range(len(dims)):
        c = rng.integers(0, 5, 48)
        c[[3, 7, 11, 19, 23, 40]] = [1, 3, 32, 33, 257, 300]
        ks.append(lay.key_base[2 * t] + np.arange(48)); cs.append(c)
    kjt = build_kjt(rng, lay, np.concatenate(ks), np.concatenate(cs), pooled=pooled)
    return lay, kjt, make_grad(rng, lay, kjt)


# =====================================================================================================================
# CPU: builder and reference
@pytest.mark.parametrize("g", [1, 2, 4, 8, 16, 32])
def test_builder_places_runs_at_requested_positions(g):
    for pooled in (True, False):
        lay, kjt, grad, placed = edge_case(g, 4 * g, pooled, n_pad=2 * (not pooled))
        pk, _ = position_keys(lay, kjt)
        order = np.argsort(pk, kind="stable")
        sk = pk[order]
        assert (np.diff(sk) >= 0).all()
        tp = tile_positions(g)
        for (key, start, length), (n, where) in zip(placed, run_specs(g)):
            assert length == n
            assert sorted_runs(lay, kjt, key) == (start, n)
            m, r = where
            assert start % m == r % m
        assert any(length == 2 * tp + 1 for _, _, length in placed)
        # padding ids sort after every real key
        if not pooled:
            assert (sk[-1000:] == 2 ** 62).all() and (sk[:-1000] < lay.total_keys).all()
        # stable: inside a run, positions ascend (pooled: ascending bag)
        brk = np.flatnonzero(np.diff(sk)) + 1
        for seg in np.split(order, brk):
            assert (np.diff(seg) > 0).all()


def test_builder_bag_lengths_and_hit_counts():
    rng = np.random.default_rng(5)
    for n in (0, 1, 3, 7, 8, 9, 1000, 600_001):
        lens = bag_lengths(rng, n)
        assert lens.sum() == n and set(np.unique(lens)) <= set(MEAN_LENS)
    lay = make_layout([(50, 8), (20, 4)], [0, 1, 0], POOL_MEAN)
    keys = np.array([0, 4, 49, 50, 69])
    counts = np.array([5, 40, 1, 300, 2])
    kjt = build_kjt(rng, lay, keys, counts, B_min=7)
    pk, feat = position_keys(lay, kjt)
    u, c = np.unique(pk, return_counts=True)
    assert np.array_equal(u, keys) and np.array_equal(c, counts)
    assert set(np.unique(feat[pk == 4])) == {0, 2}, "hits of a shared table spread over its features"
    assert len(np.unique(np.repeat(np.arange(3 * kjt.B), np.diff(kjt.offsets))[pk == 50])) > 30


@pytest.mark.parametrize("pooled", [True, False])
def test_reference_is_exact_and_order_free(pooled):
    """The float64 row sums equal fp32 sums taken in sorted order and in a random order, bit for bit."""
    lay, kjt, grad, _ = edge_case(11, 16, pooled, n_pad=0 if pooled else 3)
    gs = 0.5
    q = check_exact(lay, kjt, grad, gs)
    uk, S64 = row_sums(lay, kjt, grad, gs)
    pk, _ = position_keys(lay, kjt)
    real = pk < 2 ** 62
    srt = np.argsort(pk[real], kind="stable")
    _, S32a = row_sums(lay, kjt, grad, gs, np.float32, srt)
    _, S32b = row_sums(lay, kjt, grad, gs, np.float32, np.random.default_rng(1).permutation(int(real.sum())))
    assert np.array_equal(S32a.astype(np.float64), S64) and np.array_equal(S32b.astype(np.float64), S64)
    assert np.abs(S64).max() > 256 * q      # the long runs' sums carry many significant bits


def test_exactness_precondition_rejects_what_it_cannot_guarantee():
    lay = make_layout([(4, 4)], [0], POOL_MEAN)
    kjt = Kjt(np.zeros(3, np.int64), np.array([0, 3], np.int64), 1, True)     # a bag of 3: g / 3 is off the grid
    with pytest.raises(AssertionError):
        check_exact(lay, kjt, np.full((1, 4), Q, np.float32), 1.0)
    lay = make_layout([(4, 4)], [0], POOL_SUM)
    kjt = build_kjt(np.random.default_rng(0), lay, np.array([1]), np.array([1 << 15]), pooled=True)
    big = np.full((kjt.B, 4), 100 * Q, np.float32)                              # 2^15 * 100 * 2^-6 > 2^24 * 2^-9
    with pytest.raises(AssertionError):
        check_exact(lay, kjt, big, 1.0)


def test_hot_row_case_meets_the_precondition():
    lay, kjt, grad = hot_row_case()
    check_exact(lay, kjt, grad, 0.5)
    assert sorted_runs(lay, kjt, 5)[1] >= 600_000 and -(-600_000 // 256) > 264 * 8


def test_dispatch_mirror():
    assert dispatch(20, 4) == (8, 1) and dispatch(36, 4) == (16, 1) and dispatch(260, 4) == (32, 8)
    assert dispatch(65, 1) == (32, 8) and dispatch(256, 1) == (32, 8) and dispatch(257, 1)[1] == 9
    assert [tile_positions(g) for g in (1, 2, 4, 8, 16, 32)] == [1024, 512, 256, 128, 64, 32]


# =====================================================================================================================
# GPU
def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(params=["general", "tile"])
def path(request, monkeypatch):
    monkeypatch.setenv("TZK_BWD_TILE", "1" if request.param == "tile" else "0")
    monkeypatch.delenv("TZK_BWD_HEADS", raising=False)
    return request.param


def readout(kernels, lay, kjt, grad_t, gs=0.5):
    """SGD, lr = -1, zero arena: returns the arena (numpy float32)."""
    arena = torch.zeros(lay.arena_elems, device=DEV)
    kernels.fused_bwd(OPT_SGD, kjt.pooled, grad_t, arena, None, lay, cu(kjt.ids), cu(kjt.offsets), kjt.B, -1.0, 0.0, gs)
    torch.cuda.synchronize()
    return arena.cpu().numpy()


def assert_readout(kernels, lay, kjt, grad, gs=0.5, grad_t=None):
    check_exact(lay, kjt, grad, gs)
    uk, S = row_sums(lay, kjt, grad, gs)
    want = expected_arena(lay, uk, S.astype(np.float32))
    dlay = lay.to(DEV)
    got = readout(kernels, dlay, kjt, cu(grad) if grad_t is None else grad_t, gs)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} arena elements differ, first at {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}"
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("heads", ["heads", "walk"])
@pytest.mark.parametrize("dim", [4, 8, 16, 32, 64, 128])
@pytest.mark.parametrize("layout", ["pooled", "sequence_padded"])
def test_run_lengths_and_starts_bit_exact(kernels, monkeypatch, path, heads, dim, layout):
    """uint32 keys, VEC 4, CH 1, G = dim / 4 (1..32); general path (short runs + long-run chunk CTAs, multi-chunk
    combine) and tile path (TileCfg<G>, carry_first / carry_last, carry_combine_kernel); short-run head list
    (default) or TZK_BWD_HEADS=0.  Runs of 1, 2, 31, 32, 33, 255, 256, 257, 512, 513, TP - 1, TP, TP + 1 and 2 TP + 1
    positions, each starting at sorted positions = 0, 1, 31 (mod 32) and k TP - 1, k TP, k TP + 1.  The sequence
    layout adds zero-row padding features whose ids sort to the sentinel tail."""
    if heads == "walk":
        monkeypatch.setenv("TZK_BWD_HEADS", "0")
    pooled = layout == "pooled"
    lay, kjt, grad, _ = edge_case(zlib.crc32(f"{dim}{layout}".encode()), dim, pooled, n_pad=0 if pooled else 2)
    assert_readout(kernels, lay, kjt, grad)


def hot_row_case():
    """Row 5 of a D = 16 table hit 600 000 times: 2344 chunks of 256, more than the 264 long-run CTAs have warps."""
    rng = np.random.default_rng(600)
    lay = make_layout([(64, 16)], [0, 0], POOL_MEAN)
    keys = np.arange(64)
    counts = rng.integers(0, 40, 64)
    counts[5] = 600_000
    counts[6] = 257 * 3
    kjt = build_kjt(rng, lay, keys, counts)
    return lay, kjt, make_grad(rng, lay, kjt)


@pytest.mark.gpu
def test_hot_row_bit_exact(kernels, path):
    """uint32 keys, G 4, VEC 4, CH 1; general path: one multi-chunk run of 2344 chunks, so every long-run warp takes
    several chunk items and the last arriver combines 2344 partials in chunk order; tile path: one run over ~2300
    tiles of 256 positions (carry_combine_kernel's unrolled tile loop)."""
    lay, kjt, grad = hot_row_case()
    assert_readout(kernels, lay, kjt, grad)


DIMS = (1, 2, 3, 4, 8, 12, 16, 20, 32, 36, 64, 68, 128, 132, 256, 260, 512, 1024)


def _sweep_params():
    out = []
    for dims in [(d,) for d in DIMS] + [(4, 260), (1, 65)]:
        md = max(dims)
        natural = 4 if all(d % 4 == 0 for d in dims) else 1
        for vec in sorted({natural, 1}, reverse=True):
            g, ch = dispatch(md, vec)
            paths = ["general", "tile"] if (vec == 4 and ch == 1) else ["general"]
            for p in paths:
                tag = "x".join(map(str, dims))
                out.append(pytest.param(dims, vec, p, id=f"d{tag}-G{g}-V{vec}-CH{ch}-{p}"))
    return out


def misaligned_grad(grad, offset=1, pad=2):
    """The same values as a column slice starting at column `offset` of a wider buffer: the pointer is one float off
    16 B and ld_grad = cols + offset + pad is odd, so the kernel must take VEC 1."""
    rows, cols = grad.shape
    buf = torch.full((rows, cols + offset + pad), float("nan"), device=DEV)
    buf[:, offset:offset + cols] = cu(grad)
    view = buf[:, offset:offset + cols]
    assert view.data_ptr() % 16 != 0 and view.stride(0) % 4 != 0
    return view


@pytest.mark.gpu
@pytest.mark.parametrize("dims,vec,bwd", _sweep_params())
def test_every_lane_group_and_chunk_count(kernels, monkeypatch, dims, vec, bwd):
    """Every (G, VEC, CH) of the general path, and the tile path where it applies (VEC 4, CH 1); uint32 keys, head
    list.  VEC is 4 where every dim is a multiple of 4, and VEC 1 otherwise or when forced by a grad_out that is a
    column slice at column 1 with an odd ld_grad.  (4, 260) and (1, 65) mix a narrow feature that leaves most lanes
    idle with a wide one.  Past G 32 x CH 8 x VEC the row is rejected with the "unaligned wide rows" error."""
    monkeypatch.setenv("TZK_BWD_TILE", "1" if bwd == "tile" else "0")
    lay, kjt, grad = sweep_case(zlib.crc32(str(dims).encode()), dims)
    g, ch = dispatch(max(dims), vec)
    grad_t = misaligned_grad(grad) if vec == 1 else cu(grad)
    if ch > 8:
        dlay = lay.to(DEV)
        with pytest.raises(TzkError, match="unaligned wide rows"):
            readout(kernels, dlay, kjt, grad_t)
        return
    assert_readout(kernels, lay, kjt, grad, grad_t=grad_t)


@pytest.mark.gpu
def test_unaligned_257_is_rejected(kernels):
    """VEC 1 (D = 257 is not a multiple of 4): 257 chunks need CH 9 > 8 -> error, nothing runs."""
    lay, kjt, grad = sweep_case(257, (257,))
    arena = torch.zeros(lay.arena_elems, device=DEV)
    dlay = lay.to(DEV)
    with pytest.raises(TzkError, match="unaligned wide rows"):
        kernels.fused_bwd(OPT_SGD, True, cu(grad), arena, None, dlay, cu(kjt.ids), cu(kjt.offsets), kjt.B, -1.0, 0.0, 1.0)
    assert float(arena.abs().sum()) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [16, 64])
def test_vec1_by_alignment_matches_vec4_bit_for_bit(kernels, dim):
    """General path, uint32 keys, G = dim / 4 at VEC 4 against G = dim at VEC 1 (dim 64 -> G 32, CH 2): (a) the
    readout through a grad_out column slice at column 1 with an odd ld_grad; (b) Adagrad with a state that starts one
    float off 16 B, weights and state compared with the VEC 4 run bit for bit."""
    lay, kjt, grad = sweep_case(dim + 1, (dim,))
    v4 = assert_readout(kernels, lay, kjt, grad)
    v1 = assert_readout(kernels, lay, kjt, grad, grad_t=misaligned_grad(grad))
    assert np.array_equal(v4, v1)
    rng = np.random.default_rng(dim)
    w0 = (rng.standard_normal(lay.arena_elems) * 0.1).astype(np.float32)
    s0 = (rng.random(lay.arena_elems) * 0.01).astype(np.float32)
    dlay = lay.to(DEV)
    res = []
    for off in (0, 1):
        arena = cu(w0)
        sbuf = torch.zeros(lay.arena_elems + 4, device=DEV)
        state = sbuf[off:off + lay.arena_elems]
        state.copy_(cu(s0))
        assert (state.data_ptr() % 16 == 0) == (off == 0)
        kernels.fused_bwd(OPT_ADAGRAD, True, cu(grad), arena, state, dlay, cu(kjt.ids), cu(kjt.offsets), kjt.B,
                          2.0 ** -4, 2.0 ** -20, 0.5)
        res.append((arena.cpu().numpy(), state.cpu().numpy()))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    uk, S = row_sums(lay, kjt, grad, 0.5)
    check_update(OPT_ADAGRAD, lay, uk, S, w0, s0, None, res[0][0], res[0][1], None, dict(lr=2.0 ** -4, eps=2.0 ** -20))


# ---- uint64 keys ----------------------------------------------------------------------------------------------------
def wide_key_case(kind):
    """'big_table': a table declared with 2^32 + 7 rows of which the arena stores the first 64 -> total_keys >= 2^32
    with small keys.  'high_base': a second table whose key base is above 2^32.  'max_u32': total_keys = 2^32 - 1,
    the widest uint32 sort, with the touched rows at the very top of the key range."""
    rng = np.random.default_rng(zlib.crc32(kind.encode()))
    D = 16
    if kind == "big_table":
        lay = make_layout([(KEY32 + 7, D), (40, D)], [0, 1, 0], POOL_MEAN, stored=[64, 40])
        keys = np.concatenate([np.arange(64), KEY32 + 7 + np.arange(40)])
    elif kind == "high_base":
        lay = make_layout([(KEY32 + 7, D), (40, D)], [0, 1, 1], POOL_MEAN, stored=[64, 40])
        keys = np.concatenate([np.arange(64), KEY32 + 7 + np.arange(40)])
    else:
        lay = make_layout([(KEY32 - 1 - 40, D), (40, D)], [0, 1, 1], POOL_MEAN, stored=[64, 40])
        keys = np.concatenate([np.arange(64), KEY32 - 1 - 40 + np.arange(40)])
    counts = rng.integers(0, 6, len(keys))
    counts[[3, 70, 80]] = [300, 33, 600]
    kjt = build_kjt(rng, lay, keys, counts)
    return lay, kjt, make_grad(rng, lay, kjt)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["big_table", "high_base", "max_u32"])
def test_wide_keys_bit_exact(kernels, path, kind):
    """uint64 keys ('big_table', 'high_base'; total_keys >= 2^32) and the widest uint32 sort ('max_u32'); G 4, VEC 4,
    CH 1; general and tile path; short, single-chunk and multi-chunk runs on both tables."""
    lay, kjt, grad = wide_key_case(kind)
    assert (lay.total_keys >= KEY32) == (kind != "max_u32")
    assert_readout(kernels, lay, kjt, grad)


# ---- many features ----------------------------------------------------------------------------------------------------
def many_features_case(F, pooled):
    rng = np.random.default_rng(F)
    lay = make_layout([(3, 4)] * F, list(range(F)), POOL_MEAN if pooled else POOL_SUM)
    keys = np.arange(3 * F)
    counts = rng.integers(0, 4, 3 * F)
    counts[[1, 3 * F - 2]] = [40, 300]
    kjt = build_kjt(rng, lay, keys, counts, pooled=pooled)
    return lay, kjt, make_grad(rng, lay, kjt)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1300, 2048])
@pytest.mark.parametrize("pooled", [True, False])
def test_many_features_bit_exact(kernels, path, F, pooled):
    """uint32 keys, G 1, VEC 4, CH 1; F * sizeof(BwdFeat) > 48 KB: the feature table takes opt-in dynamic shared
    memory in fused_apply_kernel, tile_update_kernel and carry_combine_kernel (and linearize_seq_kernel for the
    sequence layout); general and tile path."""
    lay, kjt, grad = many_features_case(F, pooled)
    assert_readout(kernels, lay, kjt, grad)


@pytest.mark.gpu
def test_too_many_features_is_rejected(kernels):
    lay, kjt, grad = many_features_case(2049, True)
    dlay = lay.to(DEV)
    with pytest.raises(TzkError, match="2048"):
        readout(kernels, dlay, kjt, cu(grad))


# ---- split calls ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["hot_row", "multi_chunk_d260"])
def test_split_sort_apply_and_replay(kernels, path, case):
    """fused_bwd_sort + fused_bwd_apply give the bits of fused_bwd; a second, different gradient applied after the same
    sort is right too (multi-chunk runs reset run_done for replay).  hot_row: G 4, VEC 4, CH 1 (general or tile);
    multi_chunk_d260: G 32, VEC 4, CH 8, general path."""
    if case == "hot_row":
        lay, kjt, grad = hot_row_case()
    else:
        if path == "tile":
            pytest.skip("D = 260 runs on the general path only")
        lay, kjt, grad = sweep_case(260, (260,))
    whole = assert_readout(kernels, lay, kjt, grad)
    dlay = lay.to(DEV)
    n = len(kjt.ids)
    ws = torch.empty(kernels.fused_bwd_workspace_bytes(dlay, n), dtype=torch.uint8, device=DEV)
    kernels.fused_bwd_sort(True, dlay, cu(kjt.ids), cu(kjt.offsets), kjt.B, ws)
    grad2 = make_grad(np.random.default_rng(99), lay, kjt)
    for g in (grad, grad2):
        arena = torch.zeros(lay.arena_elems, device=DEV)
        kernels.fused_bwd_apply(OPT_SGD, True, cu(g), arena, None, dlay, cu(kjt.offsets), n, kjt.B, -1.0, 0.0, 0.5, ws)
        got = arena.cpu().numpy()
        check_exact(lay, kjt, g, 0.5)
        uk, S = row_sums(lay, kjt, g, 0.5)
        assert np.array_equal(got, expected_arena(lay, uk, S.astype(np.float32)))
        if g is grad:
            assert np.array_equal(got, whole)


# ---- optimizer math on exact row sums -------------------------------------------------------------------------------
def fp32(x):
    return float(np.float32(x))


def reference_update(opt, g, w, s, s2, rs, p):
    """float64 update of one row from its exact gradient sum `g` (after clipping), fp32 inputs.  rs: the row-wise
    state entry (row-wise Adagrad: accumulator, partial row-wise Adam: second moment).  Mirrors apply_update /
    rowwise_denom of csrc/tzk_bwd.cu."""
    lr, eps = p["lr"], p["eps"]
    if p.get("max_gradient", 0.0) > 0:
        g = np.clip(g, -p["max_gradient"], p["max_gradient"])
    b1, b2, wd, t = p.get("beta1", 0.0), p.get("beta2", 0.0), p.get("weight_decay", 0.0), p.get("t", 1)
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    if opt == OPT_SGD:
        return w - lr * g, s, s2, rs
    if opt == OPT_ADAGRAD:
        s = s + g * g
        return w - lr * g / (np.sqrt(s) + eps), s, s2, rs
    if opt == OPT_ROWWISE_ADAGRAD:
        rs = rs + np.sum(g * g) / len(g)
        return w - lr * g / (np.sqrt(rs) + eps), s, s2, rs
    m = b1 * s + (1 - b1) * g
    if opt == OPT_ADAM:
        s2 = b2 * s2 + (1 - b2) * g * g
        den = np.sqrt(s2 / bc2) + eps
    else:
        rs = b2 * rs + (1 - b2) * np.sum(g * g) / len(g)
        den = np.sqrt(rs / bc2) + eps
    return w - lr * ((m / bc1) / den + wd * w), m, s2, rs


def ulp_budget(opt, dim, vec):
    """Bound on the kernel's fp32 update error, in units of u = 2^-24 of |w| + |dw| (states: of |state|).  Each fp32
    operation of apply_update rounds once (u), __fdividef is within 2 ulp, powf within 4 ulp of beta^t, which
    1 - beta^t magnifies by beta^t / (1 - beta^t) <= 1.3 for beta <= 0.75 at t = 2.  The longest chain (Adam: m, v,
    two bias corrections, sqrt, + eps, /, + wd w, * lr, w -) stays below 20 u; 32 leaves room.  The row-wise variants
    add the fp32 sum of the row's squares: CH x VEC sequential terms per lane and a log2 G tree (<= 1 u each), halved
    by the square root."""
    if opt in (OPT_ROWWISE_ADAGRAD, OPT_PARTIAL_ROWWISE_ADAM):
        g, ch = dispatch(dim, vec)
        return 32 + (ch * vec + int(np.log2(g)) + 2) / 2
    return 32


def check_update(opt, lay, uk, S, w0, s0, s20, w, s, s2, p, rs0=None, rs=None, vec=4):
    """Compares the arena (and the states) with reference_update row by row; untouched rows must be unchanged."""
    want_w, want_s, want_s2 = w0.astype(np.float64), None if s0 is None else s0.astype(np.float64), \
        None if s20 is None else s20.astype(np.float64)
    tol_w = np.zeros(len(w0))
    tol_s = np.zeros(len(w0))
    want_rs = None if rs0 is None else rs0.astype(np.float64)
    tol_rs = None if rs0 is None else np.zeros(len(rs0))
    budget = ulp_budget(opt, lay.max_dim, vec) * U
    done = set()
    for f in range(lay.num_features):
        kb, d = lay.key_base[f], lay.dim[f]
        if lay.rows[f] == 0 or (kb, lay.w_off[f]) in done:
            continue
        done.add((kb, lay.w_off[f]))
        sel = np.flatnonzero((uk >= kb) & (uk < kb + lay.rows[f]))
        for i in sel:
            k = int(uk[i])
            o = lay.w_off[f] + (k - kb) * d
            sl = slice(o, o + d)
            nw, ns, ns2, nrs = reference_update(
                opt, S[i, :d], w0[sl].astype(np.float64), None if s0 is None else s0[sl].astype(np.float64),
                None if s20 is None else s20[sl].astype(np.float64), None if rs0 is None else float(rs0[k]), p)
            tol_w[sl] = budget * (np.abs(nw) + np.abs(nw - w0[sl]))
            want_w[sl] = nw
            if ns is not None and s0 is not None:
                want_s[sl] = ns
                tol_s[sl] = budget * np.abs(ns)
            if ns2 is not None and s20 is not None:
                want_s2[sl] = ns2
            if nrs is not None and rs0 is not None:
                want_rs[k] = nrs
                tol_rs[k] = budget * abs(nrs)
    err = np.abs(w.astype(np.float64) - want_w)
    assert (err <= tol_w).all(), f"weights: max err/tol {np.max(err / np.maximum(tol_w, 1e-300)):.3g}"
    if s0 is not None and s is not None:
        assert (np.abs(s - want_s) <= tol_s).all(), "first state"
    if s20 is not None and s2 is not None:
        assert (np.abs(s2 - want_s2) <= budget * np.abs(want_s2)).all(), "second state"
    if rs0 is not None:
        assert (np.abs(rs - want_rs) <= tol_rs).all(), "row-wise state"


OPTS = {"sgd": OPT_SGD, "adagrad": OPT_ADAGRAD, "rowwise_adagrad": OPT_ROWWISE_ADAGRAD, "adam": OPT_ADAM,
        "partial_rowwise_adam": OPT_PARTIAL_ROWWISE_ADAM}


def run_optimizer(kernels, opt, lay, kjt, grad, p, seed=0, state_keys=None):
    """One fused_bwd call on random fp32 weights and states (a row-wise state of `state_keys` entries, default
    total_keys); returns inputs and outputs as numpy arrays."""
    rng = np.random.default_rng(seed)
    dlay = lay.to(DEV)
    w0 = (rng.standard_normal(lay.arena_elems) * 0.25).astype(np.float32)
    s0 = s20 = rs0 = None
    ex = {}
    if opt in (OPT_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
        s0 = ((rng.random(lay.arena_elems) * 0.02) if opt == OPT_ADAGRAD else
              rng.standard_normal(lay.arena_elems) * 0.01).astype(np.float32)
    if opt == OPT_ADAM:
        s20 = (rng.random(lay.arena_elems) * 0.01).astype(np.float32)
    if opt in (OPT_ROWWISE_ADAGRAD, OPT_PARTIAL_ROWWISE_ADAM):
        rs0 = (rng.random(state_keys or lay.total_keys) * 0.01).astype(np.float32)
    state = cu(s0) if s0 is not None else (cu(rs0) if opt == OPT_ROWWISE_ADAGRAD else None)
    if opt == OPT_ADAM:
        ex["state2"] = cu(s20)
    if opt == OPT_PARTIAL_ROWWISE_ADAM:
        ex["state2"] = cu(rs0)
    if opt in (OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
        ex.update(step=torch.full((), float(p["t"]), device=DEV), beta1=p["beta1"], beta2=p["beta2"],
                  weight_decay=p["weight_decay"])
    if p.get("max_gradient", 0.0) > 0:
        ex["max_gradient"] = p["max_gradient"]
    arena = cu(w0)
    kernels.fused_bwd(opt, kjt.pooled, cu(grad), arena, state, dlay, cu(kjt.ids),
                      cu(kjt.offsets), kjt.B, p["lr"], p["eps"], p["gs"], **ex)
    w = arena.cpu().numpy()
    out = dict(w0=w0, w=w, s0=s0, s20=s20, rs0=rs0, s=None, s2=None, rs=None)
    if s0 is not None:
        out["s"] = state.cpu().numpy()
    if opt == OPT_ADAM:
        out["s2"] = ex["state2"].cpu().numpy()
    if opt == OPT_ROWWISE_ADAGRAD:
        out["rs"] = state.cpu().numpy()
    if opt == OPT_PARTIAL_ROWWISE_ADAM:
        out["rs"] = ex["state2"].cpu().numpy()
    return out


OPT_PARAMS = dict(lr=2.0 ** -4, eps=fp32(1e-8), gs=0.5, beta1=0.5, beta2=0.75, weight_decay=0.125, t=2)


def _opt_params():
    out = []
    for name in OPTS:
        for dims, vec, bwd in [((16,), 4, "general"), ((16,), 4, "tile"), ((128,), 4, "tile"), ((3,), 1, "general"),
                               ((68,), 4, "general"), ((260,), 4, "general"), ((1, 65), 1, "general"),
                               ((1024,), 4, "general")]:
            g, ch = dispatch(max(dims), vec)
            for clip in (0.0, 0.25):
                if clip and dims not in ((16,), (260,)):
                    continue
                tag = "x".join(map(str, dims))
                out.append(pytest.param(name, dims, bwd, clip, id=f"{name}-d{tag}-G{g}-V{vec}-CH{ch}-{bwd}"
                                                                     + ("-clip" if clip else "")))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,dims,bwd,clip", _opt_params())
def test_optimizer_math_on_exact_row_sums(kernels, monkeypatch, name, dims, bwd, clip):
    """SGD, Adagrad, row-wise Adagrad, Adam and partial row-wise Adam (weight decay 0.125, bias correction at t = 2),
    with and without max_gradient, on uint32 keys with the head list: the update computed in float64 from the exact
    row sums, within ulp_budget() of |w| + |dw|.  The id names G, VEC, CH and the path."""
    monkeypatch.setenv("TZK_BWD_TILE", "1" if bwd == "tile" else "0")
    opt = OPTS[name]
    lay, kjt, grad = sweep_case(zlib.crc32(f"opt{dims}".encode()), dims)
    p = dict(OPT_PARAMS, max_gradient=clip)
    check_exact(lay, kjt, grad, p["gs"])
    uk, S = row_sums(lay, kjt, grad, p["gs"])
    r = run_optimizer(kernels, opt, lay, kjt, grad, p, seed=len(dims) * 7 + max(dims))
    vec = 4 if all(d % 4 == 0 for d in dims) else 1
    check_update(opt, lay, uk, S, r["w0"], r["s0"], r["s20"], r["w"], r["s"], r["s2"], p, r["rs0"], r["rs"], vec)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sgd", "adagrad", "adam"])
def test_optimizer_math_on_a_key_base_above_2_32(kernels, path, name):
    """uint64 keys with a key base above 2^32, G 4, VEC 4, CH 1, general and tile path.  (The row-wise variants index
    their state by key, which would need a state of 2^32 entries here: they run in the 'big_table' case instead.)"""
    lay, kjt, grad = wide_key_case("high_base")
    p = dict(OPT_PARAMS)
    uk, S = row_sums(lay, kjt, grad, p["gs"])
    r = run_optimizer(kernels, OPTS[name], lay, kjt, grad, p)
    check_update(OPTS[name], lay, uk, S, r["w0"], r["s0"], r["s20"], r["w"], r["s"], r["s2"], p)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rowwise_adagrad", "partial_rowwise_adam"])
def test_rowwise_optimizers_on_uint64_keys_with_small_keys(kernels, name):
    """uint64 keys (a table declared with 2^32 + 7 rows, so total_keys >= 2^32) whose touched keys are all below 64:
    the row-wise state, indexed by key, needs only 64 entries.  General path, G 4, VEC 4, CH 1."""
    lay = make_layout([(KEY32 + 7, 16)], [0, 0], POOL_MEAN, stored=[64])
    assert lay.total_keys >= KEY32
    rng = np.random.default_rng(3)
    counts = rng.integers(0, 5, 64)
    counts[[2, 9]] = [33, 600]
    kjt = build_kjt(rng, lay, np.arange(64), counts)
    grad = make_grad(rng, lay, kjt)
    p = dict(OPT_PARAMS)
    uk, S = row_sums(lay, kjt, grad, p["gs"])
    opt = OPTS[name]
    r = run_optimizer(kernels, opt, lay, kjt, grad, p, state_keys=64)
    check_update(opt, lay, uk, S, r["w0"], r["s0"], r["s20"], r["w"], r["s"], r["s2"], p, r["rs0"], r["rs"])


# ---- FP16 tables ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sgd", "adagrad"])
@pytest.mark.parametrize("dims", [(4,), (16,), (64,), (3,), (128,), (260,)])
def test_fp16_tables_round_to_nearest_half(kernels, name, dims):
    """FP16 arena (w_f16), general path, uint32 keys; (G, VEC, CH) from the dims: (1,4,1), (4,4,1), (16,4,1), (4,1,1),
    (32,4,1), (32,4,8).  The fp32 update of the widened row from the exact row sum, rounded to nearest half: within
    half an ulp of the stored half (plus the fp32 update bound), untouched rows unchanged."""
    opt = OPTS[name]
    lay, kjt, grad = sweep_case(zlib.crc32(f"f16{dims}".encode()), dims)
    p = dict(OPT_PARAMS)
    uk, S = row_sums(lay, kjt, grad, p["gs"])
    rng = np.random.default_rng(4)
    w0 = (rng.standard_normal(lay.arena_elems) * 0.25).astype(np.float16)
    s0 = (rng.random(lay.arena_elems) * 0.02).astype(np.float32) if opt == OPT_ADAGRAD else None
    dlay = lay.to(DEV)
    arena = cu(w0)
    state = cu(s0) if s0 is not None else None
    kernels.fused_bwd(opt, True, cu(grad), arena, state, dlay, cu(kjt.ids), cu(kjt.offsets), kjt.B, p["lr"], p["eps"],
                      p["gs"])
    w = arena.cpu().numpy()
    vec = 4 if all(d % 4 == 0 for d in dims) else 1
    want = w0.astype(np.float64)
    tol = np.zeros(len(w0))
    budget = ulp_budget(opt, lay.max_dim, vec) * U
    for i, k in enumerate(uk):
        f = next(f for f in range(lay.num_features) if lay.key_base[f] <= k < lay.key_base[f] + lay.rows[f])
        d, kb = lay.dim[f], lay.key_base[f]
        sl = slice(lay.w_off[f] + (int(k) - kb) * d, lay.w_off[f] + (int(k) - kb + 1) * d)
        nw, _, _, _ = reference_update(opt, S[i, :d], w0[sl].astype(np.float64),
                                       None if s0 is None else s0[sl].astype(np.float64), None, None, p)
        want[sl] = nw
        tol[sl] = 0.5 * np.spacing(np.abs(w[sl])).astype(np.float64) + budget * (np.abs(nw) + np.abs(nw - w0[sl]))
    err = np.abs(w.astype(np.float64) - want)
    assert (err <= tol).all(), f"max err/tol {np.max(err / np.maximum(tol, 1e-300)):.3g}"


# ---- pooled gather over the same layouts --------------------------------------------------------------------------------
def _gather_params():
    out = []
    for dims in [(d,) for d in DIMS] + [(4, 260), (1, 65)]:
        for misaligned in (False, True):
            vec = 4 if all(d % 4 == 0 for d in dims) and not misaligned else 1
            g = dispatch(max(dims), vec)[0]
            tag = "x".join(map(str, dims))
            out.append(pytest.param(dims, misaligned, id=f"d{tag}-G{g}-V{vec}" + ("-misaligned_out" if misaligned else "")))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("pool", [POOL_SUM, POOL_MEAN])
@pytest.mark.parametrize("dims,misaligned", _gather_params())
def test_pooled_gather_exact(kernels, dims, misaligned, pool):
    """tzk_pooled_gather_fwd: pick_lanes' (G, VEC) over the same dims; table values on the grid k * 2^-6, bags of
    0, 1, 2, 4, 8 ids, so SUM and MEAN pool exactly and the output equals float64 bit for bit.  misaligned_out: `out`
    is a column slice at column 1 of a buffer with an odd row pitch (VEC 1), and nothing outside the slice changes."""
    rng = np.random.default_rng(zlib.crc32(f"g{dims}{pool}".encode()))
    lay, kjt, _ = sweep_case(zlib.crc32(str(dims).encode()), dims)
    lay.pool = [pool] * lay.num_features
    w = np.zeros(lay.arena_elems, np.float32)
    for f in range(lay.num_features):
        n = lay.rows[f] * lay.dim[f]
        w[lay.w_off[f]:lay.w_off[f] + n] = grad_values(rng, n, kmax=100)
    dlay = lay.to(DEV)
    B, F = kjt.B, lay.num_features
    want = np.zeros((B, lay.total_dim))
    lens = np.diff(kjt.offsets)
    for f in range(F):
        d = lay.dim[f]
        tab = w[lay.w_off[f]:lay.w_off[f] + lay.rows[f] * d].reshape(-1, d).astype(np.float64)
        for b in range(B):
            s, e = kjt.offsets[f * B + b], kjt.offsets[f * B + b + 1]
            if e > s:
                v = tab[kjt.ids[s:e]].sum(0)
                want[b, lay.col[f]:lay.col[f] + d] = v / (e - s) if pool == POOL_MEAN else v
    out = None
    if misaligned:
        width = lay.total_dim + 2 + ((lay.total_dim + 2) % 4 == 0)        # odd-enough pitch: never a multiple of 4
        buf = torch.full((B, width), 7.0, device=DEV)
        out = buf[:, 1:1 + lay.total_dim]
        assert out.data_ptr() % 16 != 0 and out.stride(0) % 4 != 0
    got = kernels.pooled_gather_fwd(cu(w), dlay, cu(kjt.ids), cu(kjt.offsets), B, out=out)
    assert np.array_equal(got.cpu().numpy().astype(np.float64), want)
    assert lens.max() == 8
    if misaligned:
        rest = buf.cpu().numpy()
        assert (rest[:, 0] == 7.0).all() and (rest[:, 1 + lay.total_dim:] == 7.0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1300, 2048])
def test_seq_gather_many_features_exact(kernels, F):
    """tzk_seq_gather_fwd with F up to its 2048 limit: the per-feature key boundaries it stages in shared memory grow
    past 48 KB at F = 2048.  Rows are copied, so the output equals the table rows bit for bit."""
    lay, kjt, _ = many_features_case(F, False)
    rng = np.random.default_rng(F + 1)
    w = grad_values(rng, lay.arena_elems, kmax=100)
    dlay = lay.to(DEV)
    got = kernels.seq_gather_fwd(cu(w), dlay, cu(kjt.ids), cu(kjt.offsets), kjt.B).cpu().numpy()
    feat = np.repeat(np.arange(F * kjt.B) // kjt.B, np.diff(kjt.offsets))
    base = np.asarray(lay.w_off)[feat] + kjt.ids * 4
    assert np.array_equal(got, w[base[:, None] + np.arange(4)])
