"""Float64 numpy restatement of one WuKong layer (tzrec/modules/interaction.py:236-378), forward and backward.

TEST INFRASTRUCTURE.  Written from the layer's definition: F = X (X^T W_fmb), LayerNorm(n k) -> MLP (Linear + ReLU) ->
Linear to f d, LCB W^T X, residual (W_res^T X or X), LayerNorm(d) of concat(fmb, lcb) + residual.  The split into
mix / out follows the kernels (csrc/tzk_wukong.cuh) so each can be checked on its own; `layer` composes them with the
FMB MLP for the golden fixtures of the reference's own module.
"""
import numpy as np

EPS = 1e-5


def ln_fwd(z, g, b):
    mean = z.mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((z - mean) ** 2).mean(-1, keepdims=True) + EPS)
    return (z - mean) * rstd * g + b, mean[..., 0], rstd[..., 0]


def ln_bwd(z, g, dy):
    """-> dz, dgamma, dbeta (gamma / beta gradients summed over every leading axis)."""
    mean = z.mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((z - mean) ** 2).mean(-1, keepdims=True) + EPS)
    xh = (z - mean) * rstd
    gg = dy * g
    dz = rstd * (gg - gg.mean(-1, keepdims=True) - xh * (gg * xh).mean(-1, keepdims=True))
    axes = tuple(range(z.ndim - 1))
    return dz, (dy * xh).sum(axes), dy.sum(axes)


def _f64(*a):
    return [None if t is None else np.asarray(t, np.float64) for t in a]


def interaction(x, wf):
    """X (X^T W) as [B, n k]."""
    t = np.einsum("bnd,nk->bdk", x, wf)
    return np.einsum("bnd,bdk->bnk", x, t).reshape(x.shape[0], -1)


def mix_fwd(x, wf, gf, bf, wl, wr, f):
    """-> ln_f [B, n k], stats [B, 2], base [B, f + l, d]."""
    x, wf, gf, bf, wl, wr = _f64(x, wf, gf, bf, wl, wr)
    ln_f, mean, rstd = ln_fwd(interaction(x, wf), gf, bf)
    res = x if wr is None else np.einsum("nm,bnd->bmd", wr, x)
    base = res.copy()
    base[:, f:] += np.einsum("nl,bnd->bld", wl, x)
    return ln_f, np.stack([mean, rstd], -1), base


def mix_bwd(x, wf, gf, wl, wr, f, d_ln_f, d_base):
    """-> dx, dw_fmb, dgamma, dbeta, dw_lcb, dw_res (None for the identity residual)."""
    x, wf, gf, wl, wr, d_ln_f, d_base = _f64(x, wf, gf, wl, wr, d_ln_f, d_base)
    B, n, d = x.shape
    k = wf.shape[1]
    t = np.einsum("bnd,nk->bdk", x, wf)
    fm = np.einsum("bnd,bdk->bnk", x, t).reshape(B, -1)
    dfm, dg, db = ln_bwd(fm, gf, d_ln_f)
    dfm = dfm.reshape(B, n, k)
    dt = np.einsum("bnd,bnk->bdk", x, dfm)
    dx = np.einsum("bnk,bdk->bnd", dfm, t) + np.einsum("nk,bdk->bnd", wf, dt)
    dwf = np.einsum("bnd,bdk->nk", x, dt)
    dl = d_base[:, f:]
    dx += np.einsum("nl,bld->bnd", wl, dl)
    dwl = np.einsum("bnd,bld->nl", x, dl)
    if wr is None:
        dx += d_base
        dwr = None
    else:
        dx += np.einsum("nm,bmd->bnd", wr, d_base)
        dwr = np.einsum("bnd,bmd->nm", x, d_base)
    return dx, dwf, dg, db, dwl, dwr


def _z(fmb_out, base, f):
    z = base.copy()
    B, _, d = base.shape
    z[:, :f] += fmb_out.reshape(B, f, d)
    return z


def out_fwd(fmb_out, base, g, b, f):
    """-> y [B, m, d], stats [B, m, 2]."""
    fmb_out, base, g, b = _f64(fmb_out, base, g, b)
    y, mean, rstd = ln_fwd(_z(fmb_out, base, f), g, b)
    return y, np.stack([mean, rstd], -1)


def out_bwd(fmb_out, base, g, f, dy):
    """-> d_fmb_out [B, f d], d_base, dgamma, dbeta."""
    fmb_out, base, g, dy = _f64(fmb_out, base, g, dy)
    dz, dg, db = ln_bwd(_z(fmb_out, base, f), g, dy)
    return dz[:, :f].reshape(dz.shape[0], -1).copy(), dz, dg, db


def layer(sd, x, dy, f, prefix=""):
    """The whole layer with its FMB MLP (Linear + ReLU per hidden layer, then feature_out_liner) from a state dict of
    the reference's parameter names.  -> (y, dx, {parameter name: gradient})."""
    P = {k[len(prefix):]: np.asarray(v, np.float64) for k, v in sd.items() if k.startswith(prefix)}
    x, dy = _f64(x, dy)
    wr = P.get("residual_projection.weight")
    ln_f, _, base = mix_fwd(x, P["fmb.weight"], P["fmb.norm.weight"], P["fmb.norm.bias"], P["lcb.weight"], wr, f)
    hs, h, i = [], ln_f, 0
    while f"fmb.mlp.mlp.{i}.perceptron.0.weight" in P:
        hs.append(h)
        h = np.maximum(h @ P[f"fmb.mlp.mlp.{i}.perceptron.0.weight"].T + P[f"fmb.mlp.mlp.{i}.perceptron.0.bias"], 0.0)
        i += 1
    fmb_out = h @ P["fmb.feature_out_liner.weight"].T + P["fmb.feature_out_liner.bias"]
    y, _ = out_fwd(fmb_out, base, P["norm.weight"], P["norm.bias"], f)
    grads = {}
    d_fmb, d_base, grads["norm.weight"], grads["norm.bias"] = out_bwd(fmb_out, base, P["norm.weight"], f, dy)
    grads["fmb.feature_out_liner.weight"] = d_fmb.T @ h
    grads["fmb.feature_out_liner.bias"] = d_fmb.sum(0)
    dh = d_fmb @ P["fmb.feature_out_liner.weight"]
    for j in reversed(range(i)):
        w = P[f"fmb.mlp.mlp.{j}.perceptron.0.weight"]
        out = hs[j] @ w.T + P[f"fmb.mlp.mlp.{j}.perceptron.0.bias"]
        dh = dh * (out > 0)
        grads[f"fmb.mlp.mlp.{j}.perceptron.0.weight"] = dh.T @ hs[j]
        grads[f"fmb.mlp.mlp.{j}.perceptron.0.bias"] = dh.sum(0)
        dh = dh @ w
    dx, grads["fmb.weight"], grads["fmb.norm.weight"], grads["fmb.norm.bias"], grads["lcb.weight"], dwr = mix_bwd(
        x, P["fmb.weight"], P["fmb.norm.weight"], P["lcb.weight"], wr, f, dh, d_base)
    if wr is not None:
        grads["residual_projection.weight"] = dwr
    return y, dx, grads


def seeded_case(B, d, n, l, f, k, hidden, seed):
    """Parameters under the reference's names and shapes, input X [B, n, d] and upstream gradient [B, f + l, d] of one
    layer, from uniform doubles of numpy's PCG64 stream (`Generator.random`), rounded to fp32.  The golden generator
    feeds these to the reference's WuKongLayer and stores only what it computes, so the fixture holds no inputs.
    -> (state dict, x, dy)."""
    rng = np.random.default_rng(seed)

    def u(*shape, lo=-1.0, hi=1.0):
        return (lo + (hi - lo) * rng.random(shape)).astype(np.float32)

    m = f + l
    sd = {"lcb.weight": u(n, l, lo=-0.4, hi=0.4), "fmb.weight": u(n, k, lo=-0.4, hi=0.4),
          "fmb.norm.weight": u(n * k, lo=0.9, hi=1.1), "fmb.norm.bias": u(n * k, lo=-0.1, hi=0.1)}
    width = n * k
    for i, h in enumerate(hidden):
        r = 1.0 / np.sqrt(width)
        sd[f"fmb.mlp.mlp.{i}.perceptron.0.weight"] = u(h, width, lo=-r, hi=r)
        sd[f"fmb.mlp.mlp.{i}.perceptron.0.bias"] = u(h, lo=-r, hi=r)
        width = h
    r = 1.0 / np.sqrt(width)
    sd["fmb.feature_out_liner.weight"] = u(f * d, width, lo=-r, hi=r)
    sd["fmb.feature_out_liner.bias"] = u(f * d, lo=-r, hi=r)
    sd["norm.weight"] = u(d, lo=0.9, hi=1.1)
    sd["norm.bias"] = u(d, lo=-0.1, hi=0.1)
    if n != m:
        sd["residual_projection.weight"] = u(n, m, lo=-0.4, hi=0.4)
    return sd, u(B, n, d), u(B, m, d)
