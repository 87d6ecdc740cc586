"""Float64 numpy restatement of MaskNetModule (tzrec/modules/masknet.py:20-161), forward and backward.

TEST INFRASTRUCTURE.  Written from the module's definition: ln = LayerNorm_E(e); per block
h = ReLU(x_mask W1^T + b1), m = h W2^T + b2, v = feature_input * m, o = ReLU(LayerNorm_H(v W3^T + b3)); parallel
blocks see (ln, e) and are concatenated, serial block i > 0 sees (o_{i-1}, e); then the top MLP (Linear + ReLU
layers).  The fused stages (csrc/tzk_masknet.cuh) are restated on their own (mask_fwd / mask_bwd / ffn_fwd / ffn_bwd)
in the kernels' padded layout, so each can be checked alone; `module` composes the whole thing for the golden fixture
of the reference's own module.
"""
import numpy as np

EPS = 1e-5


def pad4(n):
    return (n + 3) // 4 * 4


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
    return [np.asarray(t, np.float64) for t in a]


# ---- the fused stages, in the kernels' layout: e [B, >= E], m / v / dv / dm [B, nb Ep], z / y [B, nb H] ---------------
def mask_fwd(e, m, b2, g, b, E, nb):
    """-> v [B, nb Ep] (pad columns 0), stats [B, 2]."""
    e, m, b2, g, b = _f64(e, m, b2, g, b)
    B, Ep = e.shape[0], pad4(E)
    ln, mean, rstd = ln_fwd(e[:, :E], g, b)
    v = np.zeros((B, nb * Ep))
    for i in range(nb):
        v[:, i * Ep:i * Ep + E] = ln * (m[:, i * Ep:i * Ep + E] + b2[i * E:(i + 1) * E])
    return v, np.stack([mean, rstd], 1)


def mask_bwd(e, m, b2, g, b, dv, E, nb):
    """-> dm [B, nb Ep], de [B, Ep] (pad columns 0), db2 [nb E], dgamma [E], dbeta [E]."""
    e, m, b2, g, b, dv = _f64(e, m, b2, g, b, dv)
    B, Ep = e.shape[0], pad4(E)
    ln = ln_fwd(e[:, :E], g, b)[0]
    dm = np.zeros((B, nb * Ep))
    dln = np.zeros((B, E))
    for i in range(nb):
        dvi = dv[:, i * Ep:i * Ep + E]
        dm[:, i * Ep:i * Ep + E] = dvi * ln
        dln += dvi * (m[:, i * Ep:i * Ep + E] + b2[i * E:(i + 1) * E])
    dz, dg, db = ln_bwd(e[:, :E], g, dln)
    de = np.zeros((B, Ep))
    de[:, :E] = dz
    db2 = np.concatenate([dm[:, i * Ep:i * Ep + E].sum(0) for i in range(nb)])
    return dm, de, db2, dg, db


def ffn_fwd(z, b3, g, b, nb):
    """-> y [B, nb H] = ReLU(LN_H(z_i + b3_i)), stats [B, nb, 2]."""
    z, b3, g, b = _f64(z, b3, g, b)
    B, H = z.shape[0], z.shape[1] // nb
    t = (z + b3).reshape(B, nb, H)
    y, mean, rstd = ln_fwd(t, g.reshape(nb, H), b.reshape(nb, H))
    return np.maximum(y, 0).reshape(B, nb * H), np.stack([mean, rstd], -1)


def ffn_bwd(z, b3, g, b, dy, nb):
    """-> dz [B, nb H], dgamma [nb, H], dbeta [nb, H], db3 [nb, H]."""
    z, b3, g, b, dy = _f64(z, b3, g, b, dy)
    B, H = z.shape[0], z.shape[1] // nb
    t = (z + b3).reshape(B, nb, H)
    g3, b3_ = g.reshape(nb, H), b.reshape(nb, H)
    y = ln_fwd(t, g3, b3_)[0]
    d = dy.reshape(B, nb, H) * (y > 0)
    dz = np.zeros((B, nb, H))
    dg, db = np.zeros((nb, H)), np.zeros((nb, H))
    for i in range(nb):
        dz[:, i], dg[i], db[i] = ln_bwd(t[:, i], g3[i], d[:, i])
    return dz.reshape(B, nb * H), dg, db, dz.sum(0)


# ---- the whole module ---------------------------------------------------------------------------------------------
def block_dims(E, H, nb, ratio, agg, parallel):
    """[(input_dim, aggregation_dim)] per block, by MaskBlock's rule: a non-zero ratio overrides aggregation_dim."""
    out, d = [], E
    for _ in range(nb):
        a = int(d * ratio) if ratio else agg
        out.append((d, a))
        d = d if parallel else H
    return out


def seeded_case(B, E, ratio, agg, H, nb, top, parallel, seed):
    """(state dict with the reference's names, e [B, E], dy [B, out]) from one seeded stream."""
    rng = np.random.default_rng(seed)
    sd = {"ln_emb.weight": 1.0 + 0.1 * rng.standard_normal(E), "ln_emb.bias": 0.1 * rng.standard_normal(E)}
    for i, (d, a) in enumerate(block_dims(E, H, nb, ratio, agg, parallel)):
        p = f"mask_blocks.{i}."
        for name, shape, fan in (("mask_generator.0", (a, E), E), ("mask_generator.2", (d, a), a),
                                 ("ffn.0", (H, d), d)):
            sd[p + name + ".weight"] = rng.uniform(-1, 1, shape) / np.sqrt(fan)
            sd[p + name + ".bias"] = rng.uniform(-1, 1, shape[0]) / np.sqrt(fan)
        sd[p + "ffn.1.weight"] = 1.0 + 0.1 * rng.standard_normal(H)
        sd[p + "ffn.1.bias"] = 0.1 * rng.standard_normal(H)
    d = H * nb if parallel else H
    for j, u in enumerate(top):
        sd[f"top_mlp.mlp.{j}.perceptron.0.weight"] = rng.uniform(-1, 1, (u, d)) / np.sqrt(d)
        sd[f"top_mlp.mlp.{j}.perceptron.0.bias"] = rng.uniform(-1, 1, u) / np.sqrt(d)
        d = u
    sd = {k: v.astype(np.float32) for k, v in sd.items()}
    e = rng.standard_normal((B, E)).astype(np.float32)
    dy = rng.standard_normal((B, d)).astype(np.float32)
    return sd, e, dy


def module(sd, e, dy, nb, parallel, top_layers):
    """-> (output, de, {param name: gradient}) of MaskNetModule in float64."""
    sd = {k: np.asarray(v, np.float64) for k, v in sd.items()}
    e = np.asarray(e, np.float64)
    ln, _, _ = ln_fwd(e, sd["ln_emb.weight"], sd["ln_emb.bias"])
    caches, outs = [], []
    x = ln
    for i in range(nb):
        p = f"mask_blocks.{i}."
        fin = ln if (parallel or i == 0) else outs[-1]
        h = np.maximum(e @ sd[p + "mask_generator.0.weight"].T + sd[p + "mask_generator.0.bias"], 0)
        m = h @ sd[p + "mask_generator.2.weight"].T + sd[p + "mask_generator.2.bias"]
        v = fin * m
        t = v @ sd[p + "ffn.0.weight"].T + sd[p + "ffn.0.bias"]
        y = ln_fwd(t, sd[p + "ffn.1.weight"], sd[p + "ffn.1.bias"])[0]
        o = np.maximum(y, 0)
        caches.append((fin, h, m, v, t, y))
        outs.append(o)
    x = np.concatenate(outs, -1) if parallel else outs[-1]
    acts = [x]
    for j in range(top_layers):
        x = np.maximum(x @ sd[f"top_mlp.mlp.{j}.perceptron.0.weight"].T + sd[f"top_mlp.mlp.{j}.perceptron.0.bias"], 0)
        acts.append(x)
    grads = {}
    g = np.asarray(dy, np.float64)
    for j in reversed(range(top_layers)):
        g = g * (acts[j + 1] > 0)
        grads[f"top_mlp.mlp.{j}.perceptron.0.weight"] = g.T @ acts[j]
        grads[f"top_mlp.mlp.{j}.perceptron.0.bias"] = g.sum(0)
        g = g @ sd[f"top_mlp.mlp.{j}.perceptron.0.weight"]
    H = outs[0].shape[1]
    de = np.zeros_like(e)
    dln = np.zeros_like(e)
    d_out = [g[:, i * H:(i + 1) * H] for i in range(nb)] if parallel else [None] * (nb - 1) + [g]
    for i in reversed(range(nb)):
        p = f"mask_blocks.{i}."
        fin, h, m, v, t, y = caches[i]
        dy_i = d_out[i] * (y > 0)
        dt, grads[p + "ffn.1.weight"], grads[p + "ffn.1.bias"] = ln_bwd(t, sd[p + "ffn.1.weight"], dy_i)
        grads[p + "ffn.0.weight"] = dt.T @ v
        grads[p + "ffn.0.bias"] = dt.sum(0)
        dv = dt @ sd[p + "ffn.0.weight"]
        dfin, dm = dv * m, dv * fin
        grads[p + "mask_generator.2.weight"] = dm.T @ h
        grads[p + "mask_generator.2.bias"] = dm.sum(0)
        dh = (dm @ sd[p + "mask_generator.2.weight"]) * (h > 0)
        grads[p + "mask_generator.0.weight"] = dh.T @ e
        grads[p + "mask_generator.0.bias"] = dh.sum(0)
        de += dh @ sd[p + "mask_generator.0.weight"]
        if parallel or i == 0:
            dln += dfin
        else:
            d_out[i - 1] = dfin
    dz, grads["ln_emb.weight"], grads["ln_emb.bias"] = ln_bwd(e, sd["ln_emb.weight"], dln)
    return x, de + dz, grads
