"""float64 restatement of SelfAttentionEncoder and PoolingEncoder (tzrec/modules/sequence.py) over jagged rows, one
sample at a time: only the kept rows of a sample enter its attention, so no row sees an all-masked softmax and every
gradient is finite.  The reference's padded formulation gives the same forward (its padded query rows contribute 0 after
nan_to_num, and its padded keys carry probability 0)."""
import math

import torch


def kept(lens: torch.Tensor, max_len: int) -> torch.Tensor:
    return torch.clamp_max(lens, max_len) if max_len > 0 else lens


def self_attn_pool(q, k, v, offsets, H: int, max_len: int = 0):
    """pooled [B, E] = per head sum_i sum_j softmax_j((q_i sqrt(1/hd)) . k_j) v_j over each sample's kept rows."""
    E = q.shape[1]
    hd = E // H
    B = offsets.numel() - 1
    lens = kept(offsets[1:] - offsets[:-1], max_len)
    zero = 0 * (q.sum() + k.sum() + v.sum())          # keeps every input in the graph when no sample has rows
    out = []
    for b in range(B):
        r0, L = int(offsets[b]), int(lens[b])
        if L == 0:
            out.append(torch.zeros(E, dtype=q.dtype, device=q.device) + zero)
            continue
        qh = q[r0:r0 + L].view(L, H, hd).transpose(0, 1) * math.sqrt(1.0 / hd)
        kh = k[r0:r0 + L].view(L, H, hd).transpose(0, 1)
        vh = v[r0:r0 + L].view(L, H, hd).transpose(0, 1)
        p = torch.softmax(qh @ kh.transpose(1, 2), dim=-1)        # [H, L, L]
        out.append((p @ vh).sum(1).reshape(E))
    return torch.stack(out) if out else torch.zeros(0, E, dtype=q.dtype, device=q.device) + zero


def self_attention_encoder(seq, offsets, params, H: int, max_len: int = 0):
    """SelfAttentionEncoder.forward over jagged rows seq [N, D]; params: the reference's state-dict names."""
    p = params
    E = p["_query.weight"].shape[0]
    Q = seq @ p["_query.weight"].T + p["_query.bias"]
    K = seq @ p["_key.weight"].T + p["_key.bias"]
    V = seq @ p["_value.weight"].T + p["_value.bias"]
    W, bi = p["_multihead_attn.in_proj_weight"], p["_multihead_attn.in_proj_bias"]
    q = Q @ W[:E].T + bi[:E]
    k = K @ W[E:2 * E].T + bi[E:2 * E]
    v = V @ W[2 * E:].T + bi[2 * E:]
    pooled = self_attn_pool(q, k, v, offsets, H, max_len)
    lens = offsets[1:] - offsets[:-1]
    Lk = kept(lens, max_len).to(seq.dtype)
    out = pooled @ p["_multihead_attn.out_proj.weight"].T + Lk[:, None] * p["_multihead_attn.out_proj.bias"]
    return out / torch.clamp_min(lens, 1).to(seq.dtype)[:, None]


def pooling_encoder(seq, offsets, max_len: int = 0, mean: bool = True):
    B = offsets.numel() - 1
    lens = kept(offsets[1:] - offsets[:-1], max_len)
    out = []
    for b in range(B):
        r0, L = int(offsets[b]), int(lens[b])
        s = seq[r0:r0 + L].sum(0)
        out.append(s / max(L, 1) if mean else s)
    return torch.stack(out) if out else torch.zeros(0, seq.shape[1], dtype=seq.dtype)
