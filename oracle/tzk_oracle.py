"""CPU oracle for the sparse-embedding + feature-interaction hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under torcheasyrec_b200/ may import this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it, and only as the
checker or as the timed CPU baseline — never as the product.

It is a numpy restatement of the algorithm the reference runs for this path.  The arithmetic lives in
third-party wheels that are NOT vendored in the reference (torchrec==1.7.0, fbgemm-gpu==1.7.0;
requirements/runtime.txt:25,5), so each function restates the published semantics of the
upstream operator it names ([EXT], SURVEY.md Appendix A) and cites the reference call site that reaches it.

PINNING STATUS (see DESIGN.md §5):
  * fm(), dot_interact(), dlrm_interact(), mlp towers: pinned against golden vectors produced by the
    reference's own modules (tzrec/modules/fm.py, interaction.py, mlp.py) — tests/golden/ref_*.npz, made by
    tests/golden/make_golden_from_reference.py.
  * pooled_lookup(): pinned against torch.nn.functional.embedding_bag, the kernel the reference's un-sharded
    EmbeddingBagCollection ([EXT] torchrec.modules.embedding_modules, built at tzrec/modules/embedding.py:855)
    dispatches to on CPU; fused_update(): pinned against torch.optim.SGD / torch.optim.Adagrad applied to
    the dense autograd gradient of that lookup (tests/test_oracle_pinning.py).
  * bucketize_rw(), kjt_permute(), the TW/RW dist plumbing: "parity unpinned" — the reference holds no
    golden vectors for them (SURVEY.md §8c) and fbgemm/torchrec cannot be imported here; they are checked
    through size-independent properties (round trips, W-invariance) instead.
"""

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

POOL_SUM, POOL_MEAN = 0, 1
OPT_SGD, OPT_ADAGRAD, OPT_ROWWISE_ADAGRAD, OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM = 0, 1, 2, 3, 4

f32 = np.float32


# ----------------------------------------------------------------------------------------------------
# KJT helpers ([EXT] torchrec.sparse.jagged_tensor.KeyedJaggedTensor; layout contract of
# tzrec/datasets/utils.py:299-342 and App. A.1)
# ----------------------------------------------------------------------------------------------------
def lengths_to_offsets(lengths: np.ndarray) -> np.ndarray:
    """[EXT] fbgemm::asynchronous_complete_cumsum — offsets = [0, cumsum(lengths)] as int64."""
    out = np.zeros(len(lengths) + 1, dtype=np.int64)
    np.cumsum(lengths.astype(np.int64), out=out[1:])
    return out


def _bag_of_position(offsets: np.ndarray) -> np.ndarray:
    """bag index of every id position (inverse of offsets)."""
    n_bags = len(offsets) - 1
    return np.repeat(np.arange(n_bags, dtype=np.int64), np.diff(offsets))


def _clamp_ids(ids: np.ndarray, rows: int) -> np.ndarray:
    """[EXT] fbgemm bounds_check_mode=WARNING: an out-of-range id is replaced by row 0 (App. A.9)."""
    bad = (ids < 0) | (ids >= rows)
    if bad.any():
        ids = ids.copy()
        ids[bad] = 0
    return ids


# ----------------------------------------------------------------------------------------------------
# K4: pooled lookup  (tzrec/modules/embedding.py:930 `self.ebc(sparse_feature)`; App. A.2, A.3)
# ----------------------------------------------------------------------------------------------------
def pooled_lookup(tables: Sequence[np.ndarray], feat_table: Sequence[int], feat_pool: Sequence[int],
                  ids: np.ndarray, offsets: np.ndarray, B: int) -> np.ndarray:
    """KeyedTensor values [B, sum_f D_f]: column block f = pool over bag (f,b) of tables[feat_table[f]][id].

    SUM adds rows sequentially in list order in fp32; MEAN divides by L (empty bag -> 0)."""
    F = len(feat_table)
    dims = [tables[t].shape[1] for t in feat_table]
    out = np.zeros((B, int(sum(dims))), dtype=f32)
    col = 0
    for f in range(F):
        W = tables[feat_table[f]]
        D = W.shape[1]
        s, e = offsets[f * B], offsets[(f + 1) * B]
        fid = _clamp_ids(ids[s:e], W.shape[0])
        bag = _bag_of_position(offsets[f * B:(f + 1) * B + 1] - s)
        blk = np.zeros((B, D), dtype=f32)
        np.add.at(blk, bag, W[fid])  # unbuffered, sequential in list order
        if feat_pool[f] == POOL_MEAN:
            L = np.diff(offsets[f * B:(f + 1) * B + 1]).astype(f32)
            scale = np.where(L > 0, f32(1.0) / np.maximum(L, f32(1.0)), f32(0.0)).astype(f32)
            blk = (blk * scale[:, None]).astype(f32)
        out[:, col:col + D] = blk
        col += D
    return out


def seq_lookup(tables: Sequence[np.ndarray], feat_table: Sequence[int], ids: np.ndarray, offsets: np.ndarray,
               B: int) -> np.ndarray:
    """K4-nobag (tzrec/modules/embedding.py:1301 `ec(kjt)`): [nnz, D] rows in id order (App. A.11)."""
    F = len(feat_table)
    D = tables[feat_table[0]].shape[1] if F else 1
    out = np.zeros((len(ids), D), dtype=f32)
    for f in range(F):
        W = tables[feat_table[f]]
        s, e = offsets[f * B], offsets[(f + 1) * B]
        if W.shape[0] == 0:       # padding feature: whatever is read is never used
            continue
        out[s:e] = W[_clamp_ids(ids[s:e], W.shape[0])]
    return out


# ----------------------------------------------------------------------------------------------------
# K5: fused backward + optimizer  (tzrec/main.py:774-781, tzrec/optim/optimizer_builder.py:30-97; A.10)
# ----------------------------------------------------------------------------------------------------
def fused_update(optimizer: int, tables: List[np.ndarray], states: List[Optional[np.ndarray]],
                 feat_table: Sequence[int], feat_pool: Sequence[int], ids: np.ndarray, offsets: np.ndarray, B: int,
                 grad_out: np.ndarray, lr: float, eps: float = 1e-8, grad_scale: float = 1.0,
                 pooled: bool = True, states2: Optional[List[Optional[np.ndarray]]] = None, step: int = 1,
                 beta1: float = 0.9, beta2: float = 0.999, weight_decay: float = 0.0,
                 max_gradient: float = 0.0) -> None:
    """In-place EXACT update: per touched row g = sum of its contributions (stable order), one update.

    states[t]: ADAGRAD -> array like tables[t]; ROWWISE_ADAGRAD -> [rows]; SGD -> ignored;
    ADAM / PARTIAL_ROWWISE_ADAM -> first moment like tables[t], states2[t] = second moment (like tables[t] / [rows]).
    `step` = 1-based iteration count (bias correction).  max_gradient > 0 clamps the summed row gradient
    (gradient_clipping, tzrec/protos/optimizer.proto:76-139); weight_decay as in fbgemm's Adam:
    w -= lr * (m^ / (sqrt(v^) + eps) + weight_decay * w).  Only touched rows move (lazy / sparse semantics).
    pooled=False: grad_out is [nnz, D] (sequence / EmbeddingCollection layout)."""
    F = len(feat_table)
    lr, eps, grad_scale = f32(lr), f32(eps), f32(grad_scale)
    # gather every contribution (table, row, grad row) in id order
    per_table: Dict[int, List[Tuple[np.ndarray, np.ndarray]]] = {}
    col = 0
    for f in range(F):
        t = feat_table[f]
        W = tables[t]
        D = W.shape[1]
        s, e = offsets[f * B], offsets[(f + 1) * B]
        if W.shape[0] == 0:       # zero-row feature = wire padding of the static-capacity exchange: ignored
            col += D
            continue
        fid = _clamp_ids(ids[s:e], W.shape[0])
        if pooled:
            bag = _bag_of_position(offsets[f * B:(f + 1) * B + 1] - s)
            g = grad_out[bag, col:col + D].astype(f32)
            if feat_pool[f] == POOL_MEAN:
                L = np.diff(offsets[f * B:(f + 1) * B + 1]).astype(f32)
                g = g * (grad_scale / L[bag])[:, None]
            else:
                g = g * grad_scale
        else:
            g = grad_out[s:e].astype(f32) * grad_scale
        per_table.setdefault(t, []).append((fid, g.astype(f32)))
        col += D
    for t, parts in per_table.items():
        W = tables[t]
        rows = np.concatenate([p[0] for p in parts])
        grads = np.concatenate([p[1] for p in parts], axis=0)
        order = np.argsort(rows, kind="stable")  # contributions of a row in ascending (feature, bag) order
        rows, grads = rows[order], grads[order]
        uniq, inv = np.unique(rows, return_inverse=True)
        gsum = np.zeros((len(uniq), W.shape[1]), dtype=f32)
        np.add.at(gsum, inv, grads)
        if max_gradient > 0:
            gsum = np.clip(gsum, -f32(max_gradient), f32(max_gradient)).astype(f32)
        if optimizer == OPT_SGD:
            W[uniq] = W[uniq] - lr * gsum
        elif optimizer == OPT_ADAGRAD:
            S = states[t]
            s_new = S[uniq] + gsum * gsum
            S[uniq] = s_new
            W[uniq] = W[uniq] - lr * gsum / (np.sqrt(s_new) + eps)
        elif optimizer == OPT_ROWWISE_ADAGRAD:
            S = states[t]
            s_new = S[uniq] + (gsum * gsum).sum(axis=1, dtype=f32) / f32(W.shape[1])
            S[uniq] = s_new
            W[uniq] = W[uniq] - lr * gsum / (np.sqrt(s_new) + eps)[:, None]
        elif optimizer in (OPT_ADAM, OPT_PARTIAL_ROWWISE_ADAM):
            b1, b2, wd = f32(beta1), f32(beta2), f32(weight_decay)
            bc1 = f32(1.0) - f32(np.power(np.float32(beta1), np.float32(step)))
            bc2 = f32(1.0) - f32(np.power(np.float32(beta2), np.float32(step)))
            M, V = states[t], states2[t]
            m_new = b1 * M[uniq] + (f32(1.0) - b1) * gsum
            M[uniq] = m_new
            if optimizer == OPT_ADAM:
                v_new = b2 * V[uniq] + (f32(1.0) - b2) * gsum * gsum
                V[uniq] = v_new
                denom = np.sqrt(v_new / bc2) + eps
            else:
                v_new = b2 * V[uniq] + (f32(1.0) - b2) * ((gsum * gsum).sum(axis=1, dtype=f32) / f32(W.shape[1]))
                V[uniq] = v_new
                denom = (np.sqrt(v_new / bc2) + eps)[:, None]
            W[uniq] = W[uniq] - lr * ((m_new / bc1) / denom + wd * W[uniq])
        else:
            raise ValueError(optimizer)


# ----------------------------------------------------------------------------------------------------
# K1: row-wise block bucketize  ([EXT] fbgemm::block_bucketize_sparse_features via DMP, tzrec/main.py:799; A.7)
# ----------------------------------------------------------------------------------------------------
def rw_block_size(rows: int, W: int) -> int:
    """[EXT] torchrec row-wise shard geometry: block = ceil(H / W) (last shards short / empty)."""
    return max((rows + W - 1) // W, 1)


def bucketize_rw(ids: np.ndarray, offsets: np.ndarray, F: int, B: int, W: int, feat_block: Sequence[int],
                 feat_owner: Optional[Sequence[int]] = None):
    """dest = owner + id // block, local = id - (id // block) * block (row-wise: owner 0; table-wise: block >= rows).

    Returns (out_lengths [W*F*B] int32, out_offsets [W*F*B+1], out_ids [nnz], out_pos [nnz] int32) with the
    [W][F][B] layout; ids of a bag keep their relative order (bucketize_pos=False)."""
    nnz = len(ids)
    bag = _bag_of_position(offsets)
    f_of = bag // B
    blk = np.asarray(feat_block, dtype=np.int64)[f_of] if nnz else np.zeros(0, np.int64)
    own = (np.asarray(feat_owner, dtype=np.int64)[f_of] if feat_owner is not None else np.zeros(nnz, np.int64)) \
        if nnz else np.zeros(0, np.int64)
    q = np.where(ids < 0, 0, ids // np.maximum(blk, 1)) if nnz else bag
    dest = own + q
    over = np.maximum(dest - (W - 1), 0)
    q, dest = q - over, dest - over
    out_bag = dest * (F * B) + bag  # [W][F][B] layout
    out_lengths = np.bincount(out_bag, minlength=W * F * B).astype(np.int32)
    out_offsets = lengths_to_offsets(out_lengths)
    order = np.argsort(out_bag, kind="stable")  # keeps original relative order inside a bag
    out_ids = (ids - q * blk)[order].astype(np.int64)
    out_pos = order.astype(np.int32)
    return out_lengths, out_offsets, out_ids, out_pos


def bag_grad_expand(grad_out: np.ndarray, feat_col: Sequence[int], feat_pool: Sequence[int], offsets: np.ndarray,
                    slot: np.ndarray, F: int, B: int, D: int, n_rows: int) -> np.ndarray:
    """One gradient row per id position, placed at its wire slot (sample-owner half of the sharded backward)."""
    out = np.zeros((n_rows, D), dtype=f32)
    bag = _bag_of_position(offsets)
    f_of, b_of = bag // B, bag % B
    L = np.diff(offsets).astype(f32)
    for f in range(F):
        m = f_of == f
        g = grad_out[b_of[m], feat_col[f]:feat_col[f] + D].astype(f32)
        if feat_pool[f] == POOL_MEAN:
            g = g * (f32(1.0) / L[bag[m]])[:, None]
        out[slot[m]] = g
    return out


# ----------------------------------------------------------------------------------------------------
# K2: KJT permute  ([EXT] fbgemm::permute_2D_sparse_data; A.5)
# ----------------------------------------------------------------------------------------------------
def kjt_permute(ids: np.ndarray, lengths: np.ndarray, perm: Sequence[int], B: int):
    """Segment s of the output = segment perm[s] of the input (a segment = B consecutive bags)."""
    offsets = lengths_to_offsets(lengths)
    out_len = np.concatenate([lengths[p * B:(p + 1) * B] for p in perm]) if len(perm) else lengths[:0]
    out_ids = np.concatenate([ids[offsets[p * B]:offsets[(p + 1) * B]] for p in perm]) if len(perm) else ids[:0]
    return out_ids.astype(np.int64), out_len.astype(np.int32)


# ----------------------------------------------------------------------------------------------------
# K6 / K7
# ----------------------------------------------------------------------------------------------------
def regroup(kts: Sequence[Tuple[List[str], List[int], np.ndarray]], groups: Sequence[Sequence[str]]):
    """[EXT] KeyedTensor.regroup_as_dict (tzrec/modules/embedding.py:972-976; A.13).

    kts: (keys, length_per_key, values[B, sum]) ; returns one [B, sum] array per group."""
    where = {}
    for keys, lens, vals in kts:
        c = 0
        for k, n in zip(keys, lens):
            where[k] = (vals, c, n)
            c += n
    out = []
    for g in groups:
        out.append(np.concatenate([where[k][0][:, where[k][1]:where[k][1] + where[k][2]] for k in g], axis=1))
    return out


def to_padded_dense(values: np.ndarray, offsets: np.ndarray, T: int) -> np.ndarray:
    """[EXT] JaggedTensor.to_padded_dense (tzrec/modules/embedding.py:1429,1480; A.14)."""
    B = len(offsets) - 1
    out = np.zeros((B, T, values.shape[1]), dtype=f32)
    for b in range(B):
        n = min(int(offsets[b + 1] - offsets[b]), T)
        out[b, :n] = values[offsets[b]:offsets[b] + n]
    return out


def padded_to_jagged(grad: np.ndarray, offsets: np.ndarray, nnz: int) -> np.ndarray:
    B, T, D = grad.shape
    out = np.zeros((nnz, D), dtype=f32)
    for b in range(B):
        n = min(int(offsets[b + 1] - offsets[b]), T)
        out[offsets[b]:offsets[b] + n] = grad[b, :n]
    return out


# ----------------------------------------------------------------------------------------------------
# A7: FM  (tzrec/modules/fm.py:28-42)
# ----------------------------------------------------------------------------------------------------
def fm(x: np.ndarray) -> np.ndarray:
    """x [B,N,D] -> 0.5*((sum_n x)^2 - sum_n x^2)  (fm.py:38-42)."""
    s = x.sum(axis=1, dtype=f32)
    q = (x * x).sum(axis=1, dtype=f32)
    return (f32(0.5) * (s * s - q)).astype(f32)


def fm_bwd(x: np.ndarray, dy: np.ndarray) -> np.ndarray:
    s = x.sum(axis=1, dtype=f32)
    return (dy[:, None, :] * (s[:, None, :] - x)).astype(f32)


# ----------------------------------------------------------------------------------------------------
# A9 / A10: DLRM dot interaction  (tzrec/modules/interaction.py:80-91; tzrec/models/dlrm.py:113-131)
# ----------------------------------------------------------------------------------------------------
def dot_interact(x: np.ndarray) -> np.ndarray:
    """x [B,N,D] -> strict upper triangle of x x^T, row-major (triu_indices(N,N,1)) (interaction.py:86-91)."""
    z = np.einsum("bnd,bmd->bnm", x, x).astype(f32)
    i, j = np.triu_indices(x.shape[1], k=1)
    return z[:, i, j]


def dlrm_interact(dense: Optional[np.ndarray], sparse: np.ndarray, Ns: int, D: int, copy_dense=True,
                  copy_sparse=True) -> np.ndarray:
    """dlrm.py:113-131: cat([interaction(cat([dense[:,None], sparse])), dense, sparse])."""
    B = sparse.shape[0]
    x = sparse.reshape(B, Ns, D)
    if dense is not None:
        x = np.concatenate([dense[:, None, :], x], axis=1)
    parts = [dot_interact(x)]
    if copy_dense and dense is not None:
        parts.append(dense)
    if copy_sparse:
        parts.append(sparse)
    return np.concatenate(parts, axis=1).astype(f32)


def dlrm_interact_bwd(dense: Optional[np.ndarray], sparse: np.ndarray, d_out: np.ndarray, Ns: int, D: int,
                      copy_dense=True, copy_sparse=True):
    B = sparse.shape[0]
    x = sparse.reshape(B, Ns, D)
    if dense is not None:
        x = np.concatenate([dense[:, None, :], x], axis=1)
    N = x.shape[1]
    P = N * (N - 1) // 2
    i, j = np.triu_indices(N, k=1)
    G = np.zeros((B, N, N), dtype=f32)
    G[:, i, j] = d_out[:, :P]
    S = G + G.transpose(0, 2, 1)
    dx = np.einsum("bnm,bmd->bnd", S, x).astype(f32)
    o = P
    d_dense = None
    if dense is not None:
        d_dense = dx[:, 0, :].copy()
        if copy_dense:
            d_dense += d_out[:, o:o + D]
            o += D
        d_sparse = dx[:, 1:, :].reshape(B, Ns * D).copy()
    else:
        d_sparse = dx.reshape(B, Ns * D).copy()
    if copy_sparse:
        d_sparse += d_out[:, o:o + Ns * D]
    return d_dense, d_sparse.astype(f32)


# ----------------------------------------------------------------------------------------------------
# table init ([EXT] torchrec EmbeddingBagConfig default init_fn; A.4)
# ----------------------------------------------------------------------------------------------------
def default_table_init(rows: int, dim: int, rng: np.random.Generator) -> np.ndarray:
    bound = 1.0 / np.sqrt(rows)
    return rng.uniform(-bound, bound, size=(rows, dim)).astype(f32)
