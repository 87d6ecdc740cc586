"""Reference of the layer-wise adaptive sparse optimizers and row-wise Adagrad's weight-decay modes.

TEST INFRASTRUCTURE.  A numpy restatement, in fp32 and in the kernel's operation order, of the kFamNorm updates of
csrc/tzk_bwd.cu (finish_run_norm), which restate fbgemm_gpu's split-embedding optimizer codegen ([EXT], unverified
against a real wheel: DESIGN.md §5):

  LAMB                 m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; u = (m/bc1) / (sqrt(v/bc2) + eps) + wd w
                       w -= lr (|w| / |u|) u
  PARTIAL_ROWWISE_LAMB m element-wise, v_row = b2 v_row + (1-b2) mean_d(g^2), u with sqrt(v_row/bc2); step as LAMB
  LARS_SGD             lr' = lr eta |w| / (|g| + wd |w|) ; m = momentum m + lr' (g + wd w) ; w -= m
  ROWWISE_ADAGRAD  L2  s += mean_d((g + wd w)^2) ; w = (1 - mult wd) w - mult g      mult = lr / (sqrt(s) + eps)
                   DEC s += mean_d(g^2)          ; w = (1 - lr wd) w - mult g

`ExtOracleKernels` is tests/oracle_backend.OracleKernels with these branches added to its fused update, so the CPU
model tests can step with them; every other optimizer goes to the existing oracle unchanged.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle import tzk_oracle as O
from oracle_backend import OracleKernels, _np, _tables

OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB, OPT_LARS_SGD = 5, 6, 7
WD_NONE, WD_L2, WD_DECOUPLE = 0, 1, 2
NEW_KINDS = (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB, OPT_LARS_SGD)
f32 = np.float32


def is_norm_family(optimizer: int, weight_decay: float = 0.0, weight_decay_mode: int = WD_NONE) -> bool:
    return optimizer in NEW_KINDS or (optimizer == O.OPT_ROWWISE_ADAGRAD and weight_decay_mode != WD_NONE
                                      and weight_decay != 0.0)


def row_sums(tables, feat_table, feat_pool, ids, offsets, B, grad_out, grad_scale, pooled, max_gradient):
    """{table: (touched rows, fp32 summed + clipped gradient rows)} exactly as oracle.tzk_oracle.fused_update forms
    them: contributions in (feature, bag) order, a stable sort by row, sequential fp32 adds."""
    F = len(feat_table)
    grad_scale = f32(grad_scale)
    per_table: Dict[int, List[Tuple[np.ndarray, np.ndarray]]] = {}
    col = 0
    for f in range(F):
        t = feat_table[f]
        W = tables[t]
        D = W.shape[1]
        s, e = offsets[f * B], offsets[(f + 1) * B]
        if W.shape[0] == 0:
            col += D
            continue
        fid = O._clamp_ids(ids[s:e], W.shape[0])
        if pooled:
            bag = O._bag_of_position(offsets[f * B:(f + 1) * B + 1] - s)
            g = grad_out[bag, col:col + D].astype(f32)
            if feat_pool[f] == O.POOL_MEAN:
                L = np.diff(offsets[f * B:(f + 1) * B + 1]).astype(f32)
                g = g * (grad_scale / L[bag])[:, None]
            else:
                g = g * grad_scale
        else:
            g = grad_out[s:e].astype(f32) * grad_scale
        per_table.setdefault(t, []).append((fid, g.astype(f32)))
        col += D
    out = {}
    for t, parts in per_table.items():
        rows = np.concatenate([p[0] for p in parts])
        grads = np.concatenate([p[1] for p in parts], axis=0)
        order = np.argsort(rows, kind="stable")
        rows, grads = rows[order], grads[order]
        uniq, inv = np.unique(rows, return_inverse=True)
        gsum = np.zeros((len(uniq), tables[t].shape[1]), dtype=f32)
        np.add.at(gsum, inv, grads)
        if max_gradient > 0:
            gsum = np.clip(gsum, -f32(max_gradient), f32(max_gradient)).astype(f32)
        out[t] = (uniq, gsum)
    return out


def _sumsq(x: np.ndarray) -> np.ndarray:
    return (x * x).sum(axis=1, dtype=f32)


def update_rows(optimizer: int, w: np.ndarray, g: np.ndarray, m: Optional[np.ndarray], v: Optional[np.ndarray],
                lr: float, eps: float = 1e-8, step: int = 1, beta1: float = 0.9, beta2: float = 0.999,
                weight_decay: float = 0.0, momentum: float = 0.9, eta: float = 0.001,
                weight_decay_mode: int = WD_NONE):
    """One update of the rows w [n, D] (fp32) from their summed gradients g.  m: element-wise first state (LAMB
    variants, LARS) [n, D]; v: LAMB second moment [n, D], or the row-wise state [n] (partial row-wise LAMB second
    moment, row-wise Adagrad accumulator).  Returns (w, m, v) as new arrays."""
    lr, eps, wd = f32(lr), f32(eps), f32(weight_decay)
    w, g = w.astype(f32), g.astype(f32)
    D = f32(w.shape[1])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if optimizer in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB):
            b1, b2 = f32(beta1), f32(beta2)
            bc1 = f32(1.0) - f32(np.power(f32(beta1), f32(step)))
            bc2 = f32(1.0) - f32(np.power(f32(beta2), f32(step)))
            m = b1 * m + (f32(1.0) - b1) * g
            if optimizer == OPT_LAMB:
                v = b2 * v + (f32(1.0) - b2) * g * g
                den = np.sqrt(v / bc2) + eps
            else:
                v = b2 * v + (f32(1.0) - b2) * (_sumsq(g) / D)
                den = (np.sqrt(v / bc2) + eps)[:, None]
            u = (m / bc1) / den + wd * w
            scale = lr * (np.sqrt(_sumsq(w)) / np.sqrt(_sumsq(u)))
            return (w - scale[:, None] * u).astype(f32), m.astype(f32), v.astype(f32)
        if optimizer == OPT_LARS_SGD:
            wn = np.sqrt(_sumsq(w))
            lr_r = lr * f32(eta) * wn / (np.sqrt(_sumsq(g)) + wd * wn)
            m = f32(momentum) * m + lr_r[:, None] * (g + wd * w)
            return (w - m).astype(f32), m.astype(f32), v
        if optimizer == O.OPT_ROWWISE_ADAGRAD:
            gl = g + wd * w if weight_decay_mode == WD_L2 else g
            s = v + _sumsq(gl) / D
            mult = lr / (np.sqrt(s) + eps)
            keep = f32(1.0) - mult * wd if weight_decay_mode == WD_L2 else np.full_like(mult, f32(1.0) - lr * wd)
            return (keep[:, None] * w - mult[:, None] * g).astype(f32), m, s.astype(f32)
    raise ValueError(optimizer)


def fused_update_ext(optimizer: int, tables: List[np.ndarray], states: List[Optional[np.ndarray]],
                     feat_table: Sequence[int], feat_pool: Sequence[int], ids: np.ndarray, offsets: np.ndarray, B: int,
                     grad_out: np.ndarray, lr: float, eps: float = 1e-8, grad_scale: float = 1.0, pooled: bool = True,
                     states2: Optional[List[Optional[np.ndarray]]] = None, step: int = 1, beta1: float = 0.9,
                     beta2: float = 0.999, weight_decay: float = 0.0, max_gradient: float = 0.0,
                     momentum: float = 0.9, eta: float = 0.001, weight_decay_mode: int = WD_NONE) -> None:
    """In place, like oracle.tzk_oracle.fused_update: only touched rows move.  states[t]: LAMB variants / LARS: first
    moment like tables[t]; row-wise Adagrad: [rows].  states2[t]: LAMB: like tables[t]; partial row-wise LAMB: [rows]."""
    sums = row_sums(tables, feat_table, feat_pool, ids, offsets, B, grad_out, grad_scale, pooled, max_gradient)
    kw = dict(lr=lr, eps=eps, step=step, beta1=beta1, beta2=beta2, weight_decay=weight_decay, momentum=momentum,
              eta=eta, weight_decay_mode=weight_decay_mode)
    for t, (uniq, gsum) in sums.items():
        W = tables[t]
        if optimizer == O.OPT_ROWWISE_ADAGRAD:
            m, v = None, states[t][uniq]
        else:
            m = states[t][uniq]
            v = states2[t][uniq] if optimizer in (OPT_LAMB, OPT_PARTIAL_ROWWISE_LAMB) else None
        nw, nm, nv = update_rows(optimizer, W[uniq], gsum, m, v, **kw)
        W[uniq] = nw
        if optimizer == O.OPT_ROWWISE_ADAGRAD:
            states[t][uniq] = nv
        else:
            states[t][uniq] = nm
            if nv is not None:
                states2[t][uniq] = nv


class ExtOracleKernels(OracleKernels):
    """OracleKernels whose fused update also knows LAMB, partial row-wise LAMB, LARS-SGD and row-wise Adagrad's
    weight-decay modes (the peer and small-table models of the base class route through fused_bwd)."""

    def fused_bwd(self, optimizer, pooled, grad_out, weights, state, lay, ids, offsets, B, lr, eps, grad_scale=1.0,
                  **ex):
        if not is_norm_family(optimizer, ex.get("weight_decay", 0.0), ex.get("weight_decay_mode", WD_NONE)):
            return super().fused_bwd(optimizer, pooled, grad_out, weights, state, lay, ids, offsets, B, lr, eps,
                                     grad_scale, **ex)
        tabs, ft = _tables(weights, lay)

        def views(buf, elementwise):
            out = [None] * len(tabs)
            if buf is None:
                return out
            arr = buf.numpy()
            for f in range(lay.num_features):
                t = ft[f]
                if out[t] is None:
                    if elementwise:
                        out[t] = arr[lay.w_off[f]:lay.w_off[f] + lay.rows[f] * lay.dim[f]].reshape(lay.rows[f], lay.dim[f])
                    else:
                        out[t] = arr[lay.key_base[f]:lay.key_base[f] + lay.rows[f]]
            return out

        states = views(state, optimizer != O.OPT_ROWWISE_ADAGRAD)
        states2 = views(ex.get("state2"), optimizer == OPT_LAMB)
        step = int(round(float(ex["step"]))) if ex.get("step") is not None else 1
        fused_update_ext(optimizer, tabs, states, ft, lay.pool, _np(ids), _np(offsets), B, _np(grad_out), lr, eps,
                         grad_scale, pooled=bool(pooled), states2=states2, step=step, beta1=ex.get("beta1", 0.9),
                         beta2=ex.get("beta2", 0.999), weight_decay=ex.get("weight_decay", 0.0),
                         max_gradient=ex.get("max_gradient", 0.0), momentum=ex.get("momentum", 0.9),
                         eta=ex.get("eta", 0.001), weight_decay_mode=ex.get("weight_decay_mode", WD_NONE))
