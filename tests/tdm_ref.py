"""Float64 restatement of MultiWindowDINEncoder (tzrec/modules/sequence.py) in its padded form: the sequence as
[B, T, C] with a length per sample, the attention MLP over every padded row, the mask, the pad / crop to S = sum of
the windows, the per-window sums and their division by max(min(len - cum_w, W_w), 1).  Gradients come from torch's
autograd in float64."""
import numpy as np
import torch


def pad_rows(seq, offsets, T=None):
    """Jagged rows [N, C] + offsets [B + 1] -> padded [B, T, C] (T: the longest length by default) and lengths [B]."""
    offsets = np.asarray(offsets, np.int64)
    lens = offsets[1:] - offsets[:-1]
    B, C = len(lens), seq.shape[1]
    T = int(lens.max()) if T is None and B else (T or 0)
    out = torch.zeros((B, T, C), dtype=seq.dtype)
    for b in range(B):
        n = min(int(lens[b]), T)
        out[b, :n] = seq[offsets[b]:offsets[b] + n]
    return out, torch.from_numpy(lens)


def act(x, kind, slope):
    if kind == "relu":
        return torch.relu(x)
    return torch.where(x > 0, x, slope * x)


def multiwindow_din(query, seq_padded, lengths, windows, layers, kind, lin_w, lin_b, act_w):
    """query [B, Dq], seq_padded [B, T, C], lengths [B]; layers [(W [H, K], b [H], slope [1] or None)];
    -> [B, (L + 1) C].  Every tensor float64."""
    B, T, C = seq_padded.shape
    Dq = query.shape[1]
    mask = torch.arange(T).unsqueeze(0) < lengths.unsqueeze(1)
    q = torch.nn.functional.pad(query, (0, C - Dq)) if Dq < C else query
    qs = q.unsqueeze(1).expand(-1, T, -1)
    h = torch.cat([seq_padded, qs * seq_padded, qs], dim=-1)
    for W, b, s in layers:
        h = act(h @ W.T + b, kind, s)
    z = h @ lin_w.reshape(-1, 1) + lin_b
    a = torch.where(z > 0, z, act_w * z)
    att = a * mask.unsqueeze(2) * seq_padded
    S = int(sum(windows))
    att = torch.nn.functional.pad(att, (0, 0, 0, S - T))
    cum = np.cumsum([0] + list(windows)[:-1])
    res = []
    for w, (c0, W) in enumerate(zip(cum, windows)):
        seg = att[:, c0:c0 + W].sum(dim=1)
        cnt = torch.clamp(torch.minimum(lengths - int(c0), torch.full_like(lengths, int(W))), min=1)
        res.append(seg / cnt.unsqueeze(1).to(seg.dtype))
    return torch.cat(res + [q], dim=1)


def case(seed, B, C, Dq, hidden, windows, kind, max_len, lengths=None):
    """Seeded inputs and parameters: (query [B, Dq], seq rows [N, C], offsets [B + 1], layers, lin_w, lin_b, act_w),
    float64 tensors; lengths drawn from {0, 1, U[2, max_len], max_len} unless given."""
    g = np.random.default_rng(seed)
    if lengths is None:
        kind_l = g.integers(0, 4, size=B)
        lengths = np.where(kind_l == 0, 0, np.where(kind_l == 1, 1, np.where(
            kind_l == 2, g.integers(2, max_len + 1, size=B) if max_len >= 2 else 1, max_len)))
    lengths = np.asarray(lengths, np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    N = int(offsets[-1])
    t = lambda *s, sc=1.0: torch.from_numpy(g.standard_normal(s) * sc)  # noqa: E731
    query, seq = t(B, Dq, sc=0.5), t(N, C, sc=0.5)
    layers, K = [], 3 * C
    for H in hidden:
        layers.append((t(H, K, sc=1.0 / np.sqrt(K)), t(H, sc=0.1),
                       None if kind == "relu" else torch.tensor([0.1 + 0.3 * g.random()], dtype=torch.float64)))
        K = H
    return query, seq, offsets, layers, t(K, sc=1.0 / np.sqrt(K)), t(1, sc=0.1), torch.tensor(
        [0.25 + 0.2 * g.random()], dtype=torch.float64)
