"""Model shells that consume the hot path: DLRM, DeepFM, MMoE, PLE, PEPNet, MultiTowerDIN (+ their dense blocks).

These are the callers of §8a rows A7-A10 (SURVEY.md §2 row 4): tzrec/models/{rank_model,dlrm,deepfm,mmoe,
multi_tower_din,multi_task_rank}.py and the dense blocks of tzrec/modules/{mlp,mmoe,sequence,task_tower}.py.
Dense towers stay plain PyTorch exactly as in the reference (parameter names are kept so state_dicts line up:
`dense_mlp.mlp.0.perceptron.0.weight`, ...).  The FM / dot-interaction steps are the tzk kernels.
"""

from typing import Any, Dict, List, Optional

import contextlib
import os
import struct

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import functional as Fn
from .dense_gemm import Linear as _Linear
from .batch import Batch
from .config import Message, config_to_kwargs
from .embedding_group import EmbeddingGroup
from .embedding_modules import SparseOptimizerSpec
from .features import BaseFeature
from .kernels import (OPT_ADAGRAD, OPT_ADAM, OPT_LAMB, OPT_LARS_SGD, OPT_PARTIAL_ROWWISE_ADAM, OPT_PARTIAL_ROWWISE_LAMB,
                      OPT_ROWWISE_ADAGRAD, OPT_SGD, WD_DECOUPLE, WD_L2, WD_NONE)


# --------------------------------------------------------------------------------------------------------
# dense blocks (tzrec/modules/mlp.py:20-177, activation via eval of "nn.ReLU"-style strings)
# --------------------------------------------------------------------------------------------------------
def _create_activation(act: str) -> Optional[nn.Module]:
    if not act:
        return None
    if act.startswith("nn."):
        return getattr(nn, act[3:])()
    raise ValueError(f"Unknown activation method: {act}")


class Perceptron(nn.Module):
    def __init__(self, in_features: int, out_features: int, activation: Optional[str] = "nn.ReLU",
                 use_bn: bool = False, bias: bool = True, dropout_ratio: float = 0.0, use_ln: bool = False,
                 dim: int = 2) -> None:
        super().__init__()
        if use_bn and use_ln:
            raise ValueError("Could not use_bn and use_ln at the same time in Perceptron.")
        self.perceptron = nn.Sequential(_Linear(in_features, out_features, bias=False if use_bn else bias))
        if use_bn:
            assert dim == 2, "3-D batch norm towers are out of scope"
            self.perceptron.append(nn.BatchNorm1d(out_features))
        if use_ln:
            self.perceptron.append(nn.LayerNorm(out_features))
        if activation:
            self.perceptron.append(_create_activation(activation))
        if dropout_ratio > 0.0:
            self.perceptron.append(nn.Dropout(dropout_ratio))

    def forward(self, x: torch.Tensor, in_map=None) -> torch.Tensor:
        p = self.perceptron
        if len(p) == 2 and isinstance(p[1], nn.ReLU) and x.dim() == 2:
            # Linear -> ReLU: one fused call (BF16x9 GEMM + bias/ReLU kernel; same maths, fewer passes)
            from .dense_gemm import linear

            return linear(x, p[0].weight, p[0].bias, relu=True, in_map=in_map)
        if in_map is not None:
            from .dense_gemm import linear

            x = linear(x, p[0].weight, p[0].bias, relu=False, in_map=in_map)
            for m in list(p)[1:]:
                x = m(x)
            return x
        return p(x)


class MLP(nn.Module):
    def __init__(self, in_features: int, hidden_units: List[int], bias: bool = True,
                 activation: Optional[str] = "nn.ReLU", use_bn: bool = False, dropout_ratio=None,
                 use_ln: bool = False, dim: int = 2, return_hidden_layer_feature: bool = False, **_: Any) -> None:
        super().__init__()
        self.hidden_units = list(hidden_units)
        self.return_hidden_layer_feature = return_hidden_layer_feature
        n = len(self.hidden_units)
        if dropout_ratio is None or (isinstance(dropout_ratio, list) and len(dropout_ratio) == 0):
            dropout_ratio = [0.0] * n
        elif isinstance(dropout_ratio, list):
            dropout_ratio = dropout_ratio * n if len(dropout_ratio) == 1 else dropout_ratio
            assert len(dropout_ratio) == n, "length of dropout_ratio and hidden_units must be same"
        else:
            dropout_ratio = [dropout_ratio] * n
        self.mlp = nn.ModuleList()
        for i, h in enumerate(self.hidden_units):
            self.mlp.append(Perceptron(in_features if i == 0 else self.hidden_units[i - 1], h, activation, use_bn,
                                       bias, dropout_ratio[i], use_ln, dim))

    def output_dim(self) -> int:
        return self.hidden_units[-1]

    def forward(self, x: torch.Tensor, in_map=None):
        """`in_map`: column map of a zero-padded input (see dense_gemm.linear), consumed by the first layer.  With
        return_hidden_layer_feature: {"hidden_layer<i>": output of layer i, "hidden_layer_end": the last} instead of
        the last layer's output (mlp.py:161-177)."""
        hidden = {}
        for i, layer in enumerate(self.mlp):
            x = layer(x, in_map) if (i == 0 and in_map is not None) else layer(x)
            if self.return_hidden_layer_feature:
                hidden[f"hidden_layer{i}"] = x
        if self.return_hidden_layer_feature:
            hidden["hidden_layer_end"] = x
            return hidden
        return x


class FactorizationMachine(nn.Module):
    """tzrec/modules/fm.py:16-42, computed by tzk_fm_fwd/bwd."""

    def forward(self, feature: torch.Tensor) -> torch.Tensor:
        return Fn.factorization_machine(feature)


class InteractionArch(nn.Module):
    """tzrec/modules/interaction.py:57-91, computed by tzk_dot_interact_fwd/bwd."""

    def __init__(self, feature_num: int) -> None:
        super().__init__()
        self.feature_num = feature_num

    def output_dim(self) -> int:
        return self.feature_num * (self.feature_num - 1) // 2

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        return Fn.dot_interaction(features)


class MMoEModule(nn.Module):
    """tzrec/modules/mmoe.py:21-77."""

    def __init__(self, in_features: int, expert_mlp: Dict[str, Any], num_expert: int, num_task: int,
                 gate_mlp: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        self.num_expert, self.num_task = num_expert, num_task
        self.expert_mlps = nn.ModuleList([MLP(in_features=in_features, **expert_mlp) for _ in range(num_expert)])
        gate_in = in_features
        self.has_gate_mlp = gate_mlp is not None
        if self.has_gate_mlp:
            self.gate_mlps = nn.ModuleList([MLP(in_features=in_features, **gate_mlp) for _ in range(num_task)])
            gate_in = self.gate_mlps[0].hidden_units[-1]
        self.gate_finals = nn.ModuleList([nn.Linear(gate_in, num_expert) for _ in range(num_task)])

    def output_dim(self) -> int:
        return self.expert_mlps[0].hidden_units[-1]

    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        experts = torch.stack([m(x) for m in self.expert_mlps], dim=1)
        out = []
        for i in range(self.num_task):
            g = self.gate_mlps[i](x) if self.has_gate_mlp else x
            g = F.softmax(self.gate_finals[i](g), dim=1).unsqueeze(1)
            out.append(torch.matmul(g, experts).squeeze(1))
        return out


class TaskTower(nn.Module):
    """tzrec/modules/task_tower.py:21-52."""

    def __init__(self, tower_feature_in: int, num_class: int, mlp: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        self.tower_mlp = None
        linear_in = tower_feature_in
        if mlp is not None:
            self.tower_mlp = MLP(tower_feature_in, **mlp)
            linear_in = self.tower_mlp.output_dim()
        self.linear = _Linear(linear_in, num_class)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.tower_mlp is not None:
            x = self.tower_mlp(x)
        return self.linear(x)


class DINEncoder(nn.Module):
    """tzrec/modules/sequence.py:65-128 (target attention over the padded sequence)."""

    def __init__(self, sequence_dim: int, query_dim: int, input: str, attn_mlp: Dict[str, Any],
                 max_seq_length: int = 0, **_: Any) -> None:
        super().__init__()
        if query_dim > sequence_dim:
            raise ValueError("query_dim > sequence_dim not supported yet.")
        self._query_dim, self._sequence_dim, self._max_seq_length = query_dim, sequence_dim, max_seq_length
        self.mlp = MLP(in_features=sequence_dim * 4, dim=3, **attn_mlp)
        self.linear = nn.Linear(self.mlp.hidden_units[-1], 1)
        self._q, self._s, self._l = f"{input}.query", f"{input}.sequence", f"{input}.sequence_length"

    def output_dim(self) -> int:
        return self._sequence_dim

    def forward(self, emb: Dict[str, torch.Tensor]) -> torch.Tensor:
        query, sequence, seq_len = emb[self._q], emb[self._s], emb[self._l]
        offsets = emb.get(self._s + "_offsets")
        if offsets is not None:
            # SURVEY §8f N3: the sequence rows arrive jagged ([N, Ds], sample b = rows offsets[b]..offsets[b+1]) straight
            # from the un-pooled gather: no padded [B, T, Ds] tensor, no host read of the longest length; the attention
            # MLP runs over the N real rows only (csrc/tzk_din.cu around the dense layers)
            from . import functional as Fn

            attn_in = Fn.din_attn_input(query, sequence, offsets)
            scores = self.linear(self.mlp(attn_in)).squeeze(-1)
            return Fn.jagged_softmax_weighted_sum(scores, sequence, offsets, self._max_seq_length)
        if self._max_seq_length > 0:
            seq_len = torch.clamp_max(seq_len, self._max_seq_length)
            sequence = sequence[:, : self._max_seq_length, :]
        T = sequence.size(1)
        mask = torch.arange(T, device=seq_len.device).unsqueeze(0) < seq_len.unsqueeze(1)
        if self._query_dim < self._sequence_dim:
            query = F.pad(query, (0, self._sequence_dim - self._query_dim))
        queries = query.unsqueeze(1).expand(-1, T, -1)
        attn_in = torch.cat([queries, sequence, queries - sequence, queries * sequence], dim=-1)
        attn = self.linear(self.mlp(attn_in)).transpose(1, 2)
        padding = torch.ones_like(attn) * (-(2 ** 31) + 1)
        scores = F.softmax(torch.where(mask.unsqueeze(1), attn, padding), dim=-1)
        return torch.matmul(scores, sequence).squeeze(1)


class MultiWindowDINEncoder(nn.Module):
    """tzrec/modules/sequence.py:288-367: target attention ([k, q k, q] through attn_mlp, a Linear and a PReLU) pooled
    per time window: window w sums a_t k_t over its positions [cum_w, cum_w + W_w) and divides by
    max(min(len - cum_w, W_w), 1); the output is [window_0 .. window_{L-1}, q zero-padded to C].

    Jagged rows (`<input>.sequence_offsets` present, as TDM asks its group for): one fused call each way when
    Fn.multiwindow_din_usable holds (csrc/tzk_tdm.cuh), else Fn.torch_multiwindow_din over the same rows.  The padded
    [B, T, C] form is the reference's formulation."""

    def __init__(self, sequence_dim: int, query_dim: int, input: str, windows_len: List[int],
                 attn_mlp: Dict[str, Any], **_: Any) -> None:
        super().__init__()
        self._query_dim, self._sequence_dim = query_dim, sequence_dim
        self._windows_len = [int(w) for w in windows_len]
        if query_dim > sequence_dim:
            raise ValueError("query_dim > sequence_dim not supported yet.")
        self.register_buffer("windows_len", torch.tensor(self._windows_len))
        self.register_buffer("cumsum_windows_len", torch.tensor(np.cumsum([0] + self._windows_len[:-1])))
        self._sum_windows_len = sum(self._windows_len)
        self.mlp = MLP(in_features=sequence_dim * 3, dim=3, **attn_mlp)
        self.linear = nn.Linear(self.mlp.hidden_units[-1], 1)
        self.active = nn.PReLU()
        self._q, self._s, self._l = f"{input}.query", f"{input}.sequence", f"{input}.sequence_length"

    def output_dim(self) -> int:
        return self._sequence_dim * (len(self._windows_len) + 1)

    def forward(self, emb: Dict[str, torch.Tensor]) -> torch.Tensor:
        query, sequence, seq_len = emb[self._q], emb[self._s], emb[self._l]
        offsets = emb.get(self._s + "_offsets")
        if offsets is not None:
            if Fn.multiwindow_din_usable(query, sequence, self.mlp, self._windows_len):
                return Fn.multiwindow_din(query, sequence, offsets, self.mlp, self.linear, self.active,
                                          self._windows_len)
            return Fn.torch_multiwindow_din(query, sequence, offsets, self.mlp, self.linear, self.active,
                                            self._windows_len)
        T = sequence.size(1)
        mask = torch.arange(T, device=seq_len.device).unsqueeze(0) < seq_len.unsqueeze(1)
        if self._query_dim < self._sequence_dim:
            query = F.pad(query, (0, self._sequence_dim - self._query_dim))
        queries = query.unsqueeze(1).expand(-1, T, -1)
        attn = self.active(self.linear(self.mlp(torch.cat([sequence, queries * sequence, queries], dim=-1))))
        att_sequences = attn * mask.unsqueeze(2) * sequence
        pad = F.pad(att_sequences, (0, 0, 0, self._sum_windows_len - T)).transpose(0, 1)
        result = torch.segment_reduce(pad, reduce="sum", lengths=self.windows_len, axis=0).transpose(0, 1)
        segment_length = torch.min(seq_len.unsqueeze(1) - self.cumsum_windows_len.unsqueeze(0), self.windows_len)
        result = result / torch.max(segment_length, torch.ones_like(segment_length)).unsqueeze(2)
        return torch.cat([result, query.unsqueeze(1)], dim=1).reshape(result.shape[0], -1)


class PoolingEncoder(nn.Module):
    """tzrec/modules/sequence.py:174-218: the sum, or the mean over max(min(len, max_seq_length), 1), of the first
    max_seq_length rows (0: all).  Jagged rows: tzk_jagged_pool_fwd / _bwd (csrc/tzk_seq_attn.cuh) when
    Fn.jagged_pool_usable holds, else Fn.torch_jagged_pool; the padded [B, T, D] form is the reference's formulation."""

    def __init__(self, sequence_dim: int, input: str, pooling_type: str = "mean", max_seq_length: int = 0,
                 **_: Any) -> None:
        super().__init__()
        assert pooling_type in ["sum", "mean"], "only sum|mean pooling type supported now."
        self._sequence_dim, self._pooling_type, self._max_seq_length = sequence_dim, pooling_type, max_seq_length
        self._s, self._l = f"{input}.sequence", f"{input}.sequence_length"

    def output_dim(self) -> int:
        return self._sequence_dim

    def forward(self, emb: Dict[str, torch.Tensor]) -> torch.Tensor:
        sequence = emb[self._s]
        offsets = emb.get(self._s + "_offsets")
        mean = self._pooling_type == "mean"
        if offsets is not None:
            if Fn.jagged_pool_usable(sequence):
                return Fn.jagged_pool(sequence, offsets, self._max_seq_length, mean)
            return Fn.torch_jagged_pool(sequence, offsets, self._max_seq_length, mean)
        if self._max_seq_length > 0:
            sequence = sequence[:, : self._max_seq_length, :]
        feature = torch.sum(sequence, dim=1)
        if mean:
            seq_len = emb[self._l]
            if self._max_seq_length > 0:
                seq_len = torch.clamp_max(seq_len, self._max_seq_length)
            feature = feature / torch.clamp_min(seq_len, 1).unsqueeze(1)
        return feature


def _attention_mask(sequence: torch.Tensor, num_heads: int, sequence_length: torch.Tensor) -> torch.Tensor:
    """tzrec/modules/sequence.py:34-46: [B H, T, T], True where query or key is beyond the sample's length."""
    B, T, _ = sequence.size()
    mask = torch.arange(T, device=sequence_length.device).unsqueeze(0).expand(B, T)
    mask = (mask < sequence_length.unsqueeze(1)).int()
    mask = ~(torch.multiply(mask.unsqueeze(2), mask.unsqueeze(1)).type(torch.bool))
    return mask.repeat_interleave(repeats=num_heads, dim=0)


class SelfAttentionEncoder(nn.Module):
    """tzrec/modules/sequence.py:221-285: Q / K / V Linears, an nn.MultiheadAttention over the sequence, its output rows
    summed and divided by max(len, 1).  State-dict keys are the reference's.

    Jagged rows (`<input>.sequence_offsets` present): the Linears and the three in-projections run over the N rows, the
    attention core is Fn.self_attn_pool (csrc/tzk_seq_attn.cuh) when Fn.self_attn_pool_usable holds, else
    Fn.torch_self_attn_pool, and out_proj runs once per sample after pooling:
        out = (pooled Wo^T + L_b bo) / max(len_b, 1),   L_b = min(len_b, max_seq_length)
    (the reference's padded rows give 0, not the bias, after nan_to_num; it divides by the uncropped length).  Its
    padded query rows see every key masked, so their softmax is NaN and every parameter gradient of the padded form is
    NaN whenever lengths differ in the batch; over jagged rows no row is all-masked and the gradients are finite.
    The padded [B, T, D] form (TZK_DIN_JAGGED=0) is the reference's formulation verbatim, NaN gradients included."""

    def __init__(self, sequence_dim: int, input: str, multihead_attn_dim: int, num_heads: int = 8,
                 dropout: float = 0.0, max_seq_length: int = 0, **_: Any) -> None:
        super().__init__()
        self._sequence_dim, self._max_seq_length = sequence_dim, max_seq_length
        self._num_heads, self._multihead_attn_dim, self._dropout = num_heads, multihead_attn_dim, float(dropout)
        self._head_dim = multihead_attn_dim // num_heads
        assert self._head_dim * num_heads == multihead_attn_dim, "multihead_attn_dim must be divisible by num_heads"
        self._query = nn.Linear(sequence_dim, multihead_attn_dim)
        self._key = nn.Linear(sequence_dim, multihead_attn_dim)
        self._value = nn.Linear(sequence_dim, multihead_attn_dim)
        self._multihead_attn = nn.MultiheadAttention(multihead_attn_dim, num_heads=num_heads, dropout=dropout,
                                                     batch_first=True)
        self._s, self._l = f"{input}.sequence", f"{input}.sequence_length"

    def output_dim(self) -> int:
        return self._multihead_attn_dim

    def forward(self, emb: Dict[str, torch.Tensor]) -> torch.Tensor:
        sequence = emb[self._s]
        offsets = emb.get(self._s + "_offsets")
        if offsets is not None:
            return self._jagged(sequence, offsets)
        if self._max_seq_length > 0:
            sequence = sequence[:, : self._max_seq_length, :]
        Q, K, V = self._query(sequence), self._key(sequence), self._value(sequence)
        seq_len = emb[self._l]
        attn_mask = _attention_mask(sequence, self._num_heads, seq_len)
        attn_output, _ = self._multihead_attn(Q, K, V, attn_mask=attn_mask)
        attn_output = torch.nan_to_num(attn_output, nan=0.0)
        return attn_output.sum(dim=1) / torch.clamp_min(seq_len, 1).unsqueeze(1)

    def _jagged(self, sequence: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
        mha, E, H = self._multihead_attn, self._multihead_attn_dim, self._num_heads
        w, b = mha.in_proj_weight, mha.in_proj_bias
        q = F.linear(self._query(sequence), w[:E], b[:E])
        k = F.linear(self._key(sequence), w[E:2 * E], b[E:2 * E])
        v = F.linear(self._value(sequence), w[2 * E:], b[2 * E:])
        if Fn.self_attn_pool_usable(q, H, self._dropout, self.training):
            pooled = Fn.self_attn_pool(q, k, v, offsets, H, self._max_seq_length)
        else:
            pooled = Fn.torch_self_attn_pool(q, k, v, offsets, H, self._max_seq_length, self._dropout, self.training)
        lens = offsets[1:] - offsets[:-1]
        kept = torch.clamp_max(lens, self._max_seq_length) if self._max_seq_length > 0 else lens
        out = F.linear(pooled, mha.out_proj.weight) + kept.unsqueeze(1).to(pooled.dtype) * mha.out_proj.bias
        return out / torch.clamp_min(lens, 1).unsqueeze(1).to(out.dtype)


# the encoder kinds a DEEP group's sequence_encoders may hold (simple_attention stays outside the hot-path scope)
_SEQ_ENCODERS = {"din_encoder": DINEncoder, "pooling_encoder": PoolingEncoder,
                 "self_attention_encoder": SelfAttentionEncoder, "multi_window_din_encoder": MultiWindowDINEncoder}


def _create_seq_encoder(seq_encoder_config: Message, group_total_dim: Dict[str, int]) -> nn.Module:
    """tzrec/modules/sequence.py:370-394 for the encoder kinds built here (din_encoder, pooling_encoder,
    self_attention_encoder, multi_window_din_encoder): the encoder of a DEEP group's sequence group, with query_dim /
    sequence_dim from `<input>.query` / `<input>.sequence`."""
    kind = seq_encoder_config.WhichOneof("seq_module")
    if kind not in _SEQ_ENCODERS:
        raise NotImplementedError(f"sequence encoder {kind} is outside the hot-path scope (din_encoder, "
                                  "pooling_encoder, self_attention_encoder and multi_window_din_encoder only)")
    cfg = getattr(seq_encoder_config, kind)
    kw = config_to_kwargs(cfg)
    kw.pop("name", None)
    return _SEQ_ENCODERS[kind](sequence_dim=group_total_dim[f"{cfg.input}.sequence"],
                               query_dim=group_total_dim[f"{cfg.input}.query"], **kw)


# --------------------------------------------------------------------------------------------------------
# models
# --------------------------------------------------------------------------------------------------------
class RankModel(nn.Module):
    """tzrec/models/rank_model.py:40-287 reduced to: init_input / build_input / prediction dict / the BCE loss of a
    one-logit head or the softmax cross-entropy of a num_class > 1 head."""

    def __init__(self, model_config: Message, features: List[BaseFeature], labels: List[str],
                 sample_weights: Optional[List[str]] = None, device=None, **kwargs: Any) -> None:
        super().__init__()
        self._base_model_config = model_config
        self._model_type = model_config.WhichOneof("model")
        self._model_config = getattr(model_config, self._model_type) if self._model_type else None
        self._features, self._labels = features, labels
        self._num_class = model_config.num_class
        self._label_name = labels[0] if labels else None
        self._sample_weights = sample_weights or []
        if self._sample_weights:
            raise NotImplementedError("sample_weight_fields: weighted losses (rank_model.py:264-287 div_no_nan weighting) "
                                      "are outside the hot-path scope")
        self._device = device
        self.embedding_group: Optional[EmbeddingGroup] = None
        # label_smoothing of the softmax_cross_entropy loss (None: a BCE head)
        self._ce_smoothing: Optional[float] = None
        for lc in model_config.losses:
            kind = lc.WhichOneof("loss")
            if kind not in (None, "binary_cross_entropy", "softmax_cross_entropy"):
                raise NotImplementedError(f"loss {kind} is outside the hot-path scope (BCE-with-logits and softmax "
                                          "cross-entropy only)")
            if kind == "softmax_cross_entropy":
                self._ce_smoothing = proto_float32(lc.softmax_cross_entropy.label_smoothing)

    def init_input(self) -> None:
        """rank_model.py:83-112."""
        kw = {}
        if self._model_type == "deepfm":
            kw = dict(wide_embedding_dim=self._model_config.wide_embedding_dim or None,
                      wide_init_fn=self._model_config.wide_init_fn if self._model_config.HasField("wide_init_fn") else None)
        self.embedding_group = EmbeddingGroup(self._features, list(self._base_model_config.feature_groups),
                                              device=self._device, seq_encoder_factory=_create_seq_encoder, **kw)
        # the sequence encoders of DEEP groups read their sequence rows jagged, as MultiTowerDIN's attention towers do
        # (TZK_DIN_JAGGED=0 keeps the padded [B, T, D] form)
        seq_inputs = [getattr(enc, enc.WhichOneof("seq_module")).input for fg in self._base_model_config.feature_groups
                      for enc in fg.sequence_encoders]
        if seq_inputs and os.environ.get("TZK_DIN_JAGGED", "1") != "0":
            self.embedding_group.set_jagged_for_attention(list(dict.fromkeys(seq_inputs)))

    def build_input(self, batch: Batch) -> Dict[str, torch.Tensor]:
        """rank_model.py:114-131."""
        return self.embedding_group(batch)

    def _output_to_prediction(self, output: torch.Tensor, suffix: str = "") -> Dict[str, torch.Tensor]:
        """rank_model.py:133-179: a one-logit BCE head (logits [B], probs = sigmoid), or a softmax cross-entropy head
        (logits [B, C], probs = softmax, and probs1 = probs[:, 1] when C == 2)."""
        if self._ce_smoothing is not None:
            assert self._num_class > 1, "num_class must be greater than 1 when loss type is softmax_cross_entropy"
            probs = torch.softmax(output, dim=1)
            preds = {"logits" + suffix: output, "probs" + suffix: probs}
            if self._num_class == 2:
                preds["probs1" + suffix] = probs[:, 1]
            return preds
        assert self._num_class == 1, "only binary heads (num_class=1) are in scope"
        logits = torch.squeeze(output, dim=1)
        return {"logits" + suffix: logits, "probs" + suffix: torch.sigmoid(logits)}

    def _softmax_ce(self, logits: torch.Tensor, batch: Batch) -> torch.Tensor:
        """nn.CrossEntropyLoss(mean, label_smoothing) on the first label as a class index (rank_model.py:222-224)."""
        label = batch.labels[self._label_name].to(torch.int64)
        return F.cross_entropy(logits, label, reduction="mean", label_smoothing=self._ce_smoothing)

    def loss(self, predictions: Dict[str, torch.Tensor], batch: Batch) -> Dict[str, torch.Tensor]:
        """rank_model.py:181-287: BCEWithLogitsLoss(mean) or CrossEntropyLoss(mean) on the first label."""
        tail = getattr(self, "_tail_loss", None)
        if tail is not None:                 # computed together with the tower's tail (DLRM._fused_tail)
            self._tail_loss = None
            return {"binary_cross_entropy": tail}
        if self._ce_smoothing is not None:
            return {"softmax_cross_entropy": self._softmax_ce(predictions["logits"], batch)}
        label = batch.labels[self._label_name].to(torch.float32)
        from .dense_gemm import bce_with_logits

        return {"binary_cross_entropy": bce_with_logits(predictions["logits"], label)}

    # ---- evaluation metrics (rank_model.py:289-398, model.py:207-223): `auc` and the loss means --------------------
    def _metric_heads(self):
        """[(metric configs, loss configs, label name, name suffix)]: the model's own for single-task models."""
        return [(list(self._base_model_config.metrics), list(self._base_model_config.losses), self._label_name, "")]

    def _updated_metric_heads(self):
        """The heads update_metric adds a batch to: all of them."""
        return self._metric_heads()

    def init_metric(self, device=None, process_group=None, distributed: bool = False) -> None:
        """One metric state per configured metric and loss, named as the reference names them.  `distributed`:
        compute_metric first sums the states over `process_group` (None: the default group).  Only `auc` is
        implemented; any other metric kind raises here, i.e. when evaluation is requested."""
        from .metrics import BinnedAUC, MeanLoss

        if device is None:
            device = next(p.device for p in self.parameters() if p.device.type != "meta")
        mods = {}
        for metrics, losses, _, suffix in self._metric_heads():
            for mc in metrics:
                kind = mc.WhichOneof("metric")
                if kind != "auc":
                    raise NotImplementedError(f"metric {kind}{suffix}: only auc and the loss metrics are implemented")
                if self._ce_smoothing is not None and self._num_class > 2:
                    raise ValueError(f"auc{suffix}: num_class must be at most 2 when metric type is auc "
                                     f"(got {self._num_class})")
                mods[kind + suffix] = BinnedAUC(mc.auc.thresholds, device)
            for lc in losses:
                mods[lc.WhichOneof("loss") + suffix] = MeanLoss(device)
        self._metric_modules = mods
        self._metric_sync = (process_group, bool(distributed))

    def update_metric(self, predictions: Dict[str, torch.Tensor], batch: Batch,
                      losses: Optional[Dict[str, torch.Tensor]] = None) -> None:
        """Adds one batch to every metric state (device work only, capturable)."""
        mods = self._metric_modules
        probs = "probs1" if self._ce_smoothing is not None else "probs"      # a two-class head's auc reads probs1
        for metrics, loss_cfgs, label_name, suffix in self._updated_metric_heads():
            label = batch.labels[label_name]
            for mc in metrics:
                mods[mc.WhichOneof("metric") + suffix].update(predictions[probs + suffix], label)
            if losses is not None:
                for lc in loss_cfgs:
                    name = lc.WhichOneof("loss") + suffix
                    mods[name].update(losses[name], label.size(0))

    def compute_metric(self) -> Dict[str, torch.Tensor]:
        """{name: value} of every metric (summed over the ranks first when distributed), then every state reset.
        Raises ValueError when an auc saw labels outside {0, 1} or predictions outside [0, 1]."""
        from .metrics import compute_all

        group, distributed = self._metric_sync
        return compute_all(self._metric_modules, group, distributed)

    def sparse_collections(self):
        return list(self.embedding_group.sparse_collections())

    def set_sparse_optimizer(self, spec: SparseOptimizerSpec) -> None:
        """tzrec/main.py:774-781 (frozen tables get SGD lr=0)."""
        for coll in self.sparse_collections():
            coll.set_optimizer(spec)

    def dense_parameters(self):
        sparse_ids = {id(c.weights) for c in self.sparse_collections()}
        return [p for p in self.parameters() if id(p) not in sparse_ids and p.requires_grad]


class DLRM(RankModel):
    """tzrec/models/dlrm.py:26-135."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        eg = self.embedding_group
        self._sparse_group_name = eg.group_names()[0] if len(eg.group_names()) == 1 else "sparse"
        self.dense_mlp = None
        self._dense_group_name = "dense"
        if len(eg.group_names()) > 1 and eg.has_group(self._dense_group_name):
            self.dense_mlp = MLP(eg.group_total_dim(self._dense_group_name),
                                 **config_to_kwargs(self._model_config.dense_mlp))
        sparse_dims = eg.group_feature_dims(self._sparse_group_name)
        if len(set(sparse_dims.values())) > 1:
            raise Exception(f"sparse group feature dims must be the same, but we find {set(sparse_dims.values())}")
        self._per_sparse_dim = list(sparse_dims.values())[0]
        self._sparse_num = len(sparse_dims)
        sparse_dim = eg.group_total_dim(self._sparse_group_name)
        if self.dense_mlp and self._per_sparse_dim != self.dense_mlp.output_dim():
            raise Exception("dense mlp last hidden_unit must be the same sparse feature dim")
        self._feature_num = self._sparse_num + (1 if self.dense_mlp else 0)
        self.interaction = InteractionArch(self._feature_num)
        feature_dim = self.interaction.output_dim()
        if self.dense_mlp:
            feature_dim += self.dense_mlp.output_dim()
        if self._model_config.arch_with_sparse:
            feature_dim += sparse_dim
        self.final_mlp = MLP(feature_dim, **config_to_kwargs(self._model_config.final))
        self.output_mlp = _Linear(self.final_mlp.output_dim(), self._num_class)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        # The bottom MLP only needs the raw dense features.  Running it BEFORE the lookups gives its autograd nodes
        # the lower sequence numbers, so in the backward pass the lookups' node — which launches the fused sparse
        # update on the collection's side stream — is scheduled first and the bottom-MLP backward overlaps it.
        dense_in = self._dense_group_input(batch) if self.dense_mlp else None
        # TZK_DLRM_BOTTOM_STREAM (not through a GPU validation pass yet: on with =1 / TZK_EXPERIMENTAL=1): the bottom MLP
        # runs on a stream of its own next to the KJT scan and the lookups — it needs neither — and autograd runs its
        # backward on that stream too
        side = None
        if dense_in is not None and dense_in.is_cuda:
            from .kernels import _unvalidated_switch

            if _unvalidated_switch("TZK_DLRM_BOTTOM_STREAM"):
                side = getattr(self, "_bottom_stream", None)
                if side is None:
                    side = self._bottom_stream = torch.cuda.Stream(device=dense_in.device)
        if side is not None:
            cur = torch.cuda.current_stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                dense_feat = self.dense_mlp(dense_in)
        else:
            dense_feat = self.dense_mlp(dense_in) if dense_in is not None else None
        grouped = self.build_input(batch)
        if side is not None:
            cur.wait_stream(side)
            dense_feat.record_stream(cur)
        sparse = grouped[self._sparse_group_name]
        if self.dense_mlp and dense_feat is None:
            dense_feat = self.dense_mlp(grouped[self._dense_group_name])
        fused = self._interact_wide_tail(batch, dense_feat, sparse)
        if fused is not None:
            return fused
        x = self._interact_wide(dense_feat, sparse)
        if x is not None:           # the interaction and the first final-MLP layer in one autograd node
            in_map, start = None, 1
        elif self._interact_bf16_ok(dense_feat, sparse):
            # bf16 autocast: X [B, 784] bf16 straight from the tensor-core kernel; the first final-MLP layer is
            # autocast's F.linear over it with the weight spread by in_map (dense_gemm.linear)
            from .dense_gemm import InteractBf16Fn

            x, in_map, start = InteractBf16Fn.apply(dense_feat, sparse), InteractBf16Fn.IN_MAP, 0
        else:
            # interaction + both concats of dlrm.py:113-131 in one kernel
            # the 783-wide result travels as [B, 784]: one zero column after the 351 interaction terms puts the dense
            # and sparse blocks (and every row) on 16-B boundaries -> 128-bit stores in the kernel and tensor-core
            # (align4) kernels for the first final-MLP GEMM and its dX/dW twins (dense_gemm.py pads the weight)
            x, in_map = Fn.dlrm_interaction(dense_feat, sparse, self._sparse_num, self._per_sparse_dim,
                                            with_dense=True,
                                            with_sparse=bool(self._model_config.arch_with_sparse), aligned=True)
            start = 0
        fused = self._fused_tail(batch, x, in_map, start)
        if fused is not None:
            return fused
        for i, layer in enumerate(list(self.final_mlp.mlp)[start:], start):
            x = layer(x, in_map) if (i == 0 and in_map is not None) else layer(x)
        return self._output_to_prediction(self.output_mlp(x))

    def _interact_wide(self, dense_feat: Optional[torch.Tensor], sparse: torch.Tensor) -> Optional[torch.Tensor]:
        """Output of the first final-MLP layer computed together with the interaction (dense_gemm.InteractWideFn) when
        the model has DLRM-Criteo's shape and that layer is Linear(783 -> 64) + ReLU; None otherwise."""
        from .dense_gemm import InteractWideFn, _gemm3x_lib

        if not self._interact_wide_ok(dense_feat, sparse):
            return None
        first = self.final_mlp.mlp[0].perceptron
        return InteractWideFn.apply(_gemm3x_lib(), dense_feat, sparse, first[0].weight, first[0].bias, self._WIDE_IN_MAP)

    _WIDE_IN_MAP = ((0, 0, 351), (351, 352, 432))

    def _interact_wide_ok(self, dense_feat: Optional[torch.Tensor], sparse: torch.Tensor) -> bool:
        from .dense_gemm import interact_wide_usable

        first = self.final_mlp.mlp[0].perceptron
        return bool(self._model_config.arch_with_sparse and len(first) == 2 and isinstance(first[1], nn.ReLU)
                    and interact_wide_usable(dense_feat, sparse, first[0].weight, self._sparse_num, self._per_sparse_dim))

    def _interact_wide_tail(self, batch: Batch, dense_feat: Optional[torch.Tensor], sparse: torch.Tensor):
        """Training steps where the final MLP is the wide layer of _interact_wide and the fused tail's layer (DLRM-Criteo:
        783 -> 64 -> 32): the interaction, both layers, the output layer and the loss as one autograd node
        (dense_gemm.InteractWideTailFn), whose tail kernel also does the wide layer's ReLU backward and bias gradient.
        None when _interact_wide and _fused_tail do not both apply."""
        from .dense_gemm import InteractWideTailFn, interact_wide_tail_usable

        if len(self.final_mlp.mlp) != 2 or not self._interact_wide_ok(dense_feat, sparse):
            return None
        tail = self._tail_inputs(batch, sparse)
        if tail is None or not interact_wide_tail_usable(sparse, tail[0], tail[2], tail[4]):
            return None
        first = self.final_mlp.mlp[0].perceptron[0]
        loss, logits = InteractWideTailFn.apply(dense_feat, sparse, first.weight, first.bias, self._WIDE_IN_MAP, *tail)
        self._tail_loss = loss
        return {"logits": logits, "probs": torch.sigmoid(logits)}

    def _interact_bf16_ok(self, dense_feat: Optional[torch.Tensor], sparse: torch.Tensor) -> bool:
        """DLRM-Criteo's glue under bf16 autocast (dense_gemm.InteractBf16Fn); every other shape or dtype takes the torch
        formulation of Fn.dlrm_interaction."""
        from .dense_gemm import interact_bf16_usable

        return bool(self._model_config.arch_with_sparse) and interact_bf16_usable(dense_feat, sparse, self._sparse_num,
                                                                                   self._per_sparse_dim)

    def _fused_tail(self, batch: Batch, all_feat: torch.Tensor, in_map, start: int = 0):
        """Training steps on CUDA: the last Perceptron of the final MLP, the output layer and the BCE loss as ONE kernel
        that also produces their gradients (csrc/tzk_tower_tail.cuh; 18 launches of latency-bound work on DLRM-Criteo).
        The loss is handed to `loss()` through `_tail_loss`.  Default on; TZK_FUSED_TAIL=0 keeps the layer-by-layer chain.
        fp32 only: under autocast the layers run one by one as autocast's F.linear."""
        from .dense_gemm import tower_tail_bce, tower_tail_usable

        self._tail_loss = None
        layers = list(self.final_mlp.mlp)
        tail = self._tail_inputs(batch, all_feat)
        if tail is None:
            return None
        w1, b1, w2, b2, label = tail
        if start >= len(layers):
            return None
        x = all_feat
        for i, layer in enumerate(layers[start:-1], start):
            x = layer(x, in_map) if (i == 0 and in_map is not None) else layer(x)
        if len(layers) == 1 and in_map is not None:
            return None
        if not tower_tail_usable(x, w1, w2, label):
            return None
        loss, logits = tower_tail_bce(x, w1, b1, w2, b2, label)
        self._tail_loss = loss
        return {"logits": logits, "probs": torch.sigmoid(logits)}


    def _tail_inputs(self, batch: Batch, feat: torch.Tensor):
        """(w1, b1, w2, b2, fp32 label) of the fused tail when this step can take it: a CUDA fp32 training step with
        gradients, one class, the label in the batch, and a final MLP ending in Linear -> ReLU; None otherwise."""
        layers = list(self.final_mlp.mlp)
        if (not self.training or Fn.autocast_dtype(feat) is not None or not torch.is_grad_enabled() or not feat.is_cuda or self._num_class != 1
                or not layers or self._label_name not in batch.labels or os.environ.get("TZK_FUSED_TAIL", "1") == "0"):
            return None
        last = layers[-1].perceptron
        if not (len(last) == 2 and isinstance(last[1], nn.ReLU)):     # Linear -> ReLU only (no BN / LN / dropout)
            return None
        return (last[0].weight, last[0].bias, self.output_mlp.weight, self.output_mlp.bias,
                batch.labels[self._label_name].to(torch.float32))

    def _dense_group_input(self, batch: Batch) -> Optional[torch.Tensor]:
        """[B, 13]-style input of the `dense` group when it consists of raw dense features only (the usual DLRM
        config); None -> fall back to the grouped dictionary."""
        eg = self.embedding_group
        impl = next(iter(eg.emb_impls.values())) if len(eg.emb_impls) == 1 else None
        if impl is None or not impl.has_dense:
            return None
        key = next(iter(eg.emb_impls.keys()))
        kt = batch.dense_features.get(key)
        names = impl._group_to_shared_feature_names.get(self._dense_group_name)
        if kt is None or names is None or list(kt.keys()) != list(names):
            return None
        return kt.values()


class DeepFM(RankModel):
    """tzrec/models/deepfm.py:27-108."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        eg = self.embedding_group
        self.fm = FactorizationMachine()
        fm_group = "fm" if eg.has_group("fm") else "deep"
        self._fm_feature_dims = eg.group_dims(fm_group)
        if len(set(self._fm_feature_dims)) > 1:
            raise ValueError(f"fm feature dims must be the same, but got {self._fm_feature_dims}")
        self.deep_mlp = MLP(in_features=eg.group_total_dim("deep"), **config_to_kwargs(self._model_config.deep))
        final_dim = self.deep_mlp.output_dim()
        if self._model_config.HasField("final"):
            self.final_mlp = MLP(in_features=1 + self._fm_feature_dims[0] + final_dim,
                                 **config_to_kwargs(self._model_config.final))
            final_dim = self.final_mlp.output_dim()
        self.output_mlp = _Linear(final_dim, self._num_class)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        y_wide = torch.sum(grouped["wide"], dim=1, keepdim=True)
        deep_feat = grouped["deep"]
        y_deep = self.deep_mlp(deep_feat)
        fm_feat = grouped["fm"] if self.embedding_group.has_group("fm") else deep_feat
        y_fm = self.fm(fm_feat.reshape(-1, len(self._fm_feature_dims), self._fm_feature_dims[0]))
        if self._model_config.HasField("final"):
            y = self.output_mlp(self.final_mlp(torch.cat([y_wide, y_fm, y_deep], dim=1)))
        else:
            y = y_wide + torch.sum(y_fm, dim=1, keepdim=True) + self.output_mlp(y_deep)
        return self._output_to_prediction(y)


class MultiTowerDIN(RankModel):
    """tzrec/models/multi_tower_din.py:28-104."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        eg = self.embedding_group
        self.towers = nn.ModuleDict()
        total = 0
        for tower in self._model_config.towers:
            self.towers[tower.input] = MLP(eg.group_total_dim(tower.input), **config_to_kwargs(tower.mlp))
            total += self.towers[tower.input].output_dim()
        self.din_towers = nn.ModuleList()
        for tower in (self._model_config.din_towers if self._model_type == "multi_tower_din" else []):
            g = tower.input
            enc = DINEncoder(eg.group_total_dim(f"{g}.sequence"), eg.group_total_dim(f"{g}.query"), g,
                             attn_mlp=config_to_kwargs(tower.attn_mlp))
            self.din_towers.append(enc)
            total += enc.output_dim()
        # SURVEY §8f N3: groups whose only consumer is DIN attention keep their rows jagged (TZK_DIN_JAGGED=0 restores
        # the reference's padded [B, T, D] form)
        if len(self.din_towers) and os.environ.get("TZK_DIN_JAGGED", "1") != "0":
            eg.set_jagged_for_attention([t.input for t in self._model_config.din_towers])
        final_dim = total
        if self._model_config.HasField("final"):
            self.final_mlp = MLP(in_features=total, **config_to_kwargs(self._model_config.final))
            final_dim = self.final_mlp.output_dim()
        self.output_mlp = _Linear(final_dim, self._num_class)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        outs = [mlp(grouped[k]) for k, mlp in self.towers.items()]
        outs += [din(grouped) for din in self.din_towers]
        x = torch.cat(outs, dim=-1)
        if self._model_config.HasField("final"):
            x = self.final_mlp(x)
        return self._output_to_prediction(self.output_mlp(x))


class MultiTaskRank(RankModel):
    """tzrec/models/multi_task_rank.py:25-196 for BCE towers: one prediction pair, loss, and metric head per task tower
    (suffix `_<tower_name>`).  A tower with `task_space_indicator_label` weighs its per-sample BCE as
    multi_task_rank.py:97-142 does.  What the reference honours per tower and this repo does not (sample weights,
    non-BCE losses) is refused at construction instead of silently training with plain mean BCE."""

    # losses a task tower may use: BCE-with-logits on a one-logit head, or the JRC loss on a two-class head (only the
    # models whose reference towers accept it list jrc_loss)
    _TOWER_LOSSES = ("binary_cross_entropy",)

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        for lc in model_config.losses:          # a model-level loss: only BCE, which the towers' predictions assume
            kind = lc.WhichOneof("loss")
            if kind not in (None, "binary_cross_entropy"):
                raise NotImplementedError(f"loss {kind} is outside the hot-path scope of multi-task models "
                                          "(model-level BCE-with-logits only)")
        self._task_tower_cfgs = list(self._model_config.task_towers)
        self._jrc = {}                      # tower name -> its jrc_loss config
        for cfg in self._task_tower_cfgs:
            fld = "sample_weight_name"
            if cfg._spec(fld) is not None and cfg.HasField(fld) and getattr(cfg, fld):
                raise NotImplementedError(f"task tower {cfg.tower_name}: {fld} is outside the hot-path scope")
            for lc in (cfg.losses if cfg._spec("losses") is not None else []):
                kind = lc.WhichOneof("loss")
                if kind not in (None,) + self._TOWER_LOSSES:
                    raise NotImplementedError(f"task tower {cfg.tower_name}: loss {kind} is outside the hot-path "
                                              f"scope ({', '.join(self._TOWER_LOSSES)} only)")
                if kind == "jrc_loss":
                    assert cfg.num_class == 2, f"num_class must be 2 when loss type is {kind}"
                    self._jrc[cfg.tower_name] = lc.jrc_loss

    def _multi_task_output_to_prediction(self, tower_outputs: List[torch.Tensor]) -> Dict[str, torch.Tensor]:
        """multi_task_rank.py:50-65: tower i's output under the suffix `_<tower_name>`; a JRC tower's two-class head as
        rank_model.py:156-161: logits [B, 2], probs = softmax, probs1 = probs[:, 1]."""
        preds = {}
        for cfg, out in zip(self._task_tower_cfgs, tower_outputs):
            s = f"_{cfg.tower_name}"
            if cfg.tower_name in self._jrc:
                probs = torch.softmax(out, dim=1)
                preds.update({"logits" + s: out, "probs" + s: probs, "probs1" + s: probs[:, 1]})
            else:
                preds.update(self._output_to_prediction(out, suffix=s))
        return preds

    def _metric_heads(self):
        """multi_task_rank.py:144-196: per task tower, its metrics and losses on its label, suffixed `_<tower_name>`."""
        return [(list(c.metrics), list(c.losses), c.label_name, f"_{c.tower_name}") for c in self._task_tower_cfgs]

    def update_metric(self, predictions, batch, losses=None) -> None:
        """A JRC tower's auc reads probs1_<tower> (rank_model.py:289-330)."""
        if self._jrc:
            predictions = dict(predictions)
            for name in self._jrc:
                predictions[f"probs_{name}"] = predictions[f"probs1_{name}"]
        super().update_metric(predictions, batch, losses)

    def _session_ids(self, batch: Batch, name: str) -> torch.Tensor:
        """The first id of feature `name` in the base data group per sample, 0 for an empty row (rank_model.py:247-249
        `to_padded_dense(1)[:, 0]`), by device work only."""
        from .features import BASE_DATA_GROUP

        kjt = batch.sparse_features[BASE_DATA_GROUP]
        f, B = kjt.keys().index(name), kjt.stride()
        vals = kjt.values()
        if vals.numel() == 0:
            return torch.zeros(B, dtype=torch.int64, device=vals.device)
        start = kjt.offsets()[f * B:(f + 1) * B].to(torch.int64).clamp(max=vals.numel() - 1)
        lens = kjt.lengths()[f * B:(f + 1) * B]
        return torch.where(lens > 0, vals[start].to(torch.int64), torch.zeros_like(start))

    def _jrc_loss(self, cfg, predictions, batch) -> torch.Tensor:
        """rank_model.py:244-261 + multi_task_rank.py:97-142 for a JRC tower: the mean reduction, or, when the tower has
        `weight` or `task_space_indicator_label` (multi_task_rank.py:67-78), mean(loss * w) with w =
        div_no_nan(v, mean v) * weight."""
        jc = self._jrc[cfg.tower_name]
        label = batch.labels[cfg.label_name].to(torch.float32)
        sid = self._session_ids(batch, jc.session_name)
        alpha = proto_float32(jc.alpha)
        logits = predictions[f"logits_{cfg.tower_name}"]
        w = None
        if cfg.HasField("weight") or _task_space_label(cfg):
            w = torch.ones(1, device=label.device)
            if _task_space_label(cfg):
                in_space = (batch.labels[cfg.task_space_indicator_label] > 0).float()
                w = w * (cfg.in_task_space_weight * in_space + cfg.out_task_space_weight * (1 - in_space))
            w = torch.nan_to_num(torch.div(w, torch.mean(w)), nan=0.0, posinf=0.0, neginf=0.0) * cfg.weight
        # the raw ids of the batch, not bounded by the table (the lookup clamps, the grouping must not): all 64 bits
        return Fn.jrc_loss(logits, label, sid, alpha, w)

    def loss(self, predictions, batch):
        from .dense_gemm import bce_with_logits

        out = {}
        for cfg in self._task_tower_cfgs:
            if cfg.tower_name in self._jrc:
                out[f"jrc_loss_{cfg.tower_name}"] = self._jrc_loss(cfg, predictions, batch)
                continue
            label = batch.labels[cfg.label_name].to(torch.float32)
            logits = predictions[f"logits_{cfg.tower_name}"]
            if _task_space_label(cfg):
                out[f"binary_cross_entropy_{cfg.tower_name}"] = task_space_weighted_bce(
                    logits, label, batch.labels[cfg.task_space_indicator_label], cfg.in_task_space_weight,
                    cfg.out_task_space_weight, cfg.weight)
            else:
                out[f"binary_cross_entropy_{cfg.tower_name}"] = cfg.weight * bce_with_logits(logits, label)
        return out


def _task_space_label(cfg) -> Optional[str]:
    fld = "task_space_indicator_label"
    return getattr(cfg, fld) if cfg._spec(fld) is not None and cfg.HasField(fld) and getattr(cfg, fld) else None


def task_space_weighted_bce(logits: torch.Tensor, label: torch.Tensor, indicator: torch.Tensor, in_weight: float,
                            out_weight: float, weight: float) -> torch.Tensor:
    """multi_task_rank.py:105-125 + rank_model.py:233-261 for a tower with task_space_indicator_label and no sample
    weight: mean(bce_none * w), w = div_no_nan(v, mean(v)) * weight, v = in [ind > 0] + out (1 - [ind > 0]).  Device
    work only (capturable): an all-out-of-space batch with out_weight 0 gives w = 0, not NaN."""
    logits = logits.float()
    in_space = (indicator > 0).float()
    w = torch.ones(1, device=logits.device) * (in_weight * in_space + out_weight * (1 - in_space))
    w = torch.nan_to_num(torch.div(w, torch.mean(w)), nan=0.0, posinf=0.0, neginf=0.0)
    w = w * weight
    return torch.mean(F.binary_cross_entropy_with_logits(logits, label, reduction="none") * w)


class MMoE(MultiTaskRank):
    """tzrec/models/mmoe.py:24-86 + multi_task_rank.py:50-65 (one BCE loss per tower, summed)."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        self.mmoe = MMoEModule(
            in_features=self.embedding_group.group_total_dim(self.group_name),
            expert_mlp=config_to_kwargs(self._model_config.expert_mlp), num_expert=self._model_config.num_expert,
            num_task=len(self._task_tower_cfgs),
            gate_mlp=config_to_kwargs(self._model_config.gate_mlp) if self._model_config.HasField("gate_mlp") else None)
        self._task_tower = nn.ModuleList()
        for cfg in self._task_tower_cfgs:
            mlp = config_to_kwargs(cfg.mlp) if cfg.HasField("mlp") else None
            self._task_tower.append(TaskTower(self.mmoe.output_dim(), cfg.num_class, mlp=mlp))

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        task_inputs = self.mmoe(grouped[self.group_name])
        return self._multi_task_output_to_prediction([tower(x) for tower, x in zip(self._task_tower, task_inputs)])


class ExtractionNet(nn.Module):
    """tzrec/modules/extraction_net.py:20-133: one PLE extraction layer.  `expert_num_per_task` experts per task on that
    task's input and `share_num` shared experts on the shared input (each an MLP); task gate i mixes
    [task i experts..., shared experts...], the shared gate (not in the last layer) mixes [every task expert...,
    shared experts...].  When Fn.ple_gate_usable holds, all of the layer's gates run as one fused call
    (Fn.ple_gates, csrc/tzk_ple.cuh); otherwise the reference's torch formulation."""

    def __init__(self, in_extraction_networks: List[int], in_shared_expert: int, network_name: str, share_num: int,
                 expert_num_per_task: int, share_expert_net: Dict[str, Any], task_expert_net: Dict[str, Any],
                 final_flag: bool = False) -> None:
        super().__init__()
        self.name = network_name
        self._final_flag = final_flag
        self._shared_layers = nn.ModuleList([MLP(in_shared_expert, **share_expert_net) for _ in range(share_num)])
        self._shared_gate = None
        if not final_flag:
            self._shared_gate = nn.Linear(in_shared_expert, len(in_extraction_networks) * expert_num_per_task + share_num)
        self._task_layers = nn.ModuleList()
        self._task_gates = nn.ModuleList()
        self._output_dims = []
        for in_feature in in_extraction_networks:
            self._task_layers.append(nn.ModuleList([MLP(in_feature, **task_expert_net)
                                                    for _ in range(expert_num_per_task)]))
            self._task_gates.append(nn.Linear(in_feature, expert_num_per_task + share_num))
            self._output_dims.append(task_expert_net["hidden_units"][-1])
        self._output_dims.append(share_expert_net["hidden_units"][-1])

    def output_dim(self) -> List[int]:
        return self._output_dims

    def gate_layout(self):
        """(gate_input, gate_experts) of Fn.ple_gates for the layer's experts in the order
        [task 0 experts..., task 1 experts..., ..., shared experts...]; input 0 is the shared input, input 1 + i task
        i's (the caller merges inputs that are the same tensor)."""
        T, S = len(self._task_layers), len(self._shared_layers)
        per = len(self._task_layers[0]) if T else 0
        shared = list(range(T * per, T * per + S))
        gate_input = [1 + i for i in range(T)]
        gate_experts = [list(range(i * per, (i + 1) * per)) + shared for i in range(T)]
        if self._shared_gate is not None:
            gate_input.append(0)
            gate_experts.append(list(range(T * per + S)))
        return gate_input, gate_experts

    def forward(self, extraction_network_fea: List[torch.Tensor], shared_expert_fea: torch.Tensor):
        shared_expert = [layer(shared_expert_fea) for layer in self._shared_layers]
        task_experts = [[layer(extraction_network_fea[i]) for layer in layers]
                        for i, layers in enumerate(self._task_layers)]
        experts = [e for te in task_experts for e in te] + shared_expert
        gate_input, gate_experts = self.gate_layout()
        candidates = [shared_expert_fea] + list(extraction_network_fea)
        inputs = []                       # the distinct tensors the gates read, by identity (one in the first layer)
        for i in gate_input:
            if not any(candidates[i] is u for u in inputs):
                inputs.append(candidates[i])
        gate_input = [next(j for j, u in enumerate(inputs) if u is candidates[i]) for i in gate_input]
        gates = list(self._task_gates) + ([self._shared_gate] if self._shared_gate is not None else [])
        weights = [g.weight for g in gates]
        if Fn.ple_gate_usable(inputs, gate_input, weights, experts, gate_experts):
            outs = Fn.ple_gates(inputs, gate_input, weights, [g.bias for g in gates], experts, gate_experts)
        else:
            outs = [Fn.torch_ple_gate(inputs[gate_input[g]], [experts[x] for x in gate_experts[g]], gates[g])
                    for g in range(len(gates))]
        T = len(self._task_layers)
        return outs[:T], (outs[T] if self._shared_gate is not None else None)


class PLE(MultiTaskRank):
    """tzrec/models/ple.py:26-112: the first feature group through the stacked extraction layers, then one task tower
    per task on its branch of the last layer."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self._task_nums = len(self._task_tower_cfgs)
        self._layer_nums = len(self._model_config.extraction_networks)
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        feature_in = self.embedding_group.group_total_dim(self.group_name)
        self._extraction_nets = nn.ModuleList()
        in_extraction_networks, in_shared_expert = [feature_in] * self._task_nums, feature_in
        for i, cfg in enumerate(self._model_config.extraction_networks):
            extraction = ExtractionNet(in_extraction_networks, in_shared_expert, final_flag=i == self._layer_nums - 1,
                                       **config_to_kwargs(cfg))
            self._extraction_nets.append(extraction)
            output_dims = extraction.output_dim()
            in_extraction_networks, in_shared_expert = output_dims[:-1], output_dims[-1]
        self._task_tower = nn.ModuleList()
        for i, cfg in enumerate(self._task_tower_cfgs):
            mlp = config_to_kwargs(cfg.mlp) if cfg.HasField("mlp") else None
            self._task_tower.append(TaskTower(in_extraction_networks[i], cfg.num_class, mlp=mlp))

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        net = self.build_input(batch)[self.group_name]
        extraction_network_fea, shared_expert_fea = [net] * self._task_nums, net
        for extraction_net in self._extraction_nets:
            extraction_network_fea, shared_expert_fea = extraction_net(extraction_network_fea, shared_expert_fea)
        return self._multi_task_output_to_prediction(
            [tower(x) for tower, x in zip(self._task_tower, extraction_network_fea)])


class GateNU(nn.Module):
    """tzrec/modules/personalized_net.py:20-59: gamma * sigmoid(Linear(ReLU(Linear(x))))."""

    def __init__(self, input_dim: int, hidden_dim: int, output_dim: int, gamma: float = 2.0) -> None:
        super().__init__()
        self._gamma = gamma
        self._output_dim = output_dim
        self.dense_layers = nn.Sequential(nn.Linear(input_dim, hidden_dim), nn.ReLU(), nn.Linear(hidden_dim, output_dim),
                                          nn.Sigmoid())

    def output_dim(self) -> int:
        return self._output_dim

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self._gamma * self.dense_layers(x)


class EPNet(nn.Module):
    """tzrec/modules/personalized_net.py:62-110: GateNU([domain | main.detach()]) * main.  When Fn.pepnet_usable holds,
    the gate's first layer, its second layer and the sigmoid product run as Fn.pepnet_gate_hidden +
    Fn.pepnet_product (csrc/tzk_pepnet.cuh); otherwise the reference's torch formulation."""

    def __init__(self, main_dim: int, domain_dim: int, hidden_dim: int, gamma: float = 2.0) -> None:
        super().__init__()
        self._domain_dim, self._main_dim, self._hidden_dim = domain_dim, main_dim, hidden_dim
        self.gate_nu = GateNU(input_dim=domain_dim + main_dim, hidden_dim=hidden_dim, output_dim=main_dim, gamma=gamma)

    def output_dim(self) -> int:
        return self.gate_nu.output_dim()

    def forward(self, main_emb: torch.Tensor, domain_emb: torch.Tensor) -> torch.Tensor:
        if Fn.pepnet_usable(main_emb, domain_emb, [self._hidden_dim], [self._main_dim]):
            z = Fn.pepnet_gate_hidden(domain_emb, main_emb, [self.gate_nu], [self._main_dim], [(0, 0)])[0]
            return Fn.pepnet_product(z, [self.gate_nu], self.gate_nu._gamma, [main_emb])
        gate_input = torch.cat([domain_emb, main_emb.detach()], dim=-1)
        return self.gate_nu(gate_input) * main_emb


class PPNet(nn.Module):
    """tzrec/modules/personalized_net.py:113-196: per task i and depth j (module index i * len_hidden + j),
    y_ij = Dropout(act(Linear_ij(y_i,j-1)) * GateNU_ij([uia | main.detach()])), y_i,-1 = main.  When Fn.pepnet_usable
    holds: every GateNU's first layer over all tasks and depths as one GEMM on the gate input formed once
    (Fn.pepnet_gate_hidden), then per depth one fused product over all tasks (Fn.pepnet_product; depth 0's linears as
    one GEMM of the shared input) and the reference's Dropout modules; otherwise the reference's torch formulation."""

    def __init__(self, main_feature: int, uia_feature: int, num_task: int, hidden_units: List[int],
                 activation: Optional[str] = "nn.ReLU", dropout_ratio=None, gamma: float = 2.0) -> None:
        super().__init__()
        self.main_feature, self.uia_feature, self.num_task = main_feature, uia_feature, num_task
        self.hidden_units = list(hidden_units)
        self.len_hidden = len(self.hidden_units)
        self._activation, self._gamma = activation, gamma
        self.linears = nn.ModuleList()
        self.activations = nn.ModuleList()
        self.dropout_ratios = nn.ModuleList()
        self.gate_nus = nn.ModuleList()
        n = len(self.hidden_units)
        if dropout_ratio is None:
            dropout_ratio = [0.0] * n
        elif isinstance(dropout_ratio, list):
            if len(dropout_ratio) == 0:
                dropout_ratio = [0.0] * n
            elif len(dropout_ratio) == 1:
                dropout_ratio = dropout_ratio * n
            else:
                assert len(dropout_ratio) == n, ("length of dropout_ratio and hidden_units must be same, "
                                                 f"but got {len(dropout_ratio)} vs {n}")
        else:
            dropout_ratio = [dropout_ratio] * n
        for _ in range(self.num_task):
            output = main_feature
            for i, hidden_unit in enumerate(self.hidden_units):
                self.linears.append(nn.Linear(output, hidden_unit))
                self.activations.append(_create_activation(activation))
                self.dropout_ratios.append(nn.Dropout(dropout_ratio[i]))
                self.gate_nus.append(GateNU(input_dim=main_feature + uia_feature, hidden_dim=hidden_unit,
                                            output_dim=hidden_unit, gamma=gamma))
                output = hidden_unit

    def output_dim(self) -> List[int]:
        return [self.hidden_units[-1]] * self.num_task

    def task_output_dim(self) -> int:
        return self.hidden_units[-1]

    def fused_usable(self, main_emb: torch.Tensor, uia_emb: torch.Tensor) -> bool:
        return Fn.pepnet_usable(main_emb, uia_emb, self.hidden_units, self.hidden_units, self.num_task,
                                self._activation)

    def forward(self, main_emb: torch.Tensor, uia_emb: torch.Tensor) -> List[torch.Tensor]:
        T, L = self.num_task, self.len_hidden
        if self.fused_usable(main_emb, uia_emb):
            gates = list(self.gate_nus)
            place = [(j, i * self.hidden_units[j]) for i in range(T) for j in range(L)]
            zs = Fn.pepnet_gate_hidden(uia_emb, main_emb, gates, [T * h for h in self.hidden_units], place)
            outs = [main_emb]
            for j, h in enumerate(self.hidden_units):
                ks = [i * L + j for i in range(T)]
                y = Fn.pepnet_product(zs[j], [gates[k] for k in ks], self._gamma, outs,
                                      [self.linears[k] for k in ks], relu=True)
                outs = [self.dropout_ratios[k](y[:, i * h:(i + 1) * h]) for i, k in enumerate(ks)]
            return outs
        task_outputs = []
        for i in range(T):
            gate_input = torch.cat([uia_emb, main_emb.detach()], dim=-1)
            x = main_emb
            for j in range(L):
                k = i * L + j
                x = self.linears[k](x)
                x = self.activations[k](x)
                x = x * self.gate_nus[k](gate_input)
                x = self.dropout_ratios[k](x)
            task_outputs.append(x)
        return task_outputs


def _float32(v: float) -> float:
    """A `float` proto field as the reference's model reads it straight off the message: the stored float32's value."""
    return struct.unpack("f", struct.pack("f", float(v)))[0]


class PEPNet(MultiTaskRank):
    """tzrec/models/pepnet.py:27-244: group `all` through EPNet (when a `domain` group exists) and PPNet (when a `uia`
    group exists), then the task towers; with domain_input_name, task_domain_num towers per task (`_task_tower.{i D +
    j}`) whose predictions are `logits_<tower>_<j>` / `probs_<tower>_<j>`, and the loss and the metrics see the tower
    of each sample's domain label as `logits_<tower>` / `probs_<tower>`.

    The selection is sum_j [d == j] out_j (exact; only the selected tower receives a gradient), so it never indexes
    memory with a label value: a domain label outside [0, D) selects 0 where the reference's torch.gather raises."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        eg = self.embedding_group
        self._main_group_name, self._domain_group_name, self._uia_group_name = "all", "domain", "uia"
        if not eg.has_group(self._main_group_name):
            raise Exception("all feature group not found.")
        self._main_group_dim = eg.group_total_dim(self._main_group_name)
        self._task_input_dim = self._main_group_dim
        cfg = self._model_config
        self.epnet = None
        if eg.has_group(self._domain_group_name):
            self.epnet = EPNet(self._main_group_dim, eg.group_total_dim(self._domain_group_name),
                               hidden_dim=cfg.epnet_hidden_unit if cfg.HasField("epnet_hidden_unit")
                               else self._main_group_dim, gamma=_float32(cfg.epnet_gamma))
            self._task_input_dim = self.epnet.output_dim()
        self.ppnet = None
        if eg.has_group(self._uia_group_name):
            self.ppnet = PPNet(self._main_group_dim, eg.group_total_dim(self._uia_group_name),
                               num_task=len(self._task_tower_cfgs), hidden_units=list(cfg.ppnet_hidden_units),
                               activation=cfg.ppnet_activation,
                               dropout_ratio=[_float32(r) for r in cfg.ppnet_dropout_ratio],
                               gamma=_float32(cfg.ppnet_gamma))
            self._task_input_dim = self.ppnet.task_output_dim()
        self._domain_input_name = cfg.domain_input_name if cfg.HasField("domain_input_name") else None
        self._task_domain_num = cfg.task_domain_num
        self._task_tower = nn.ModuleList()
        for tc in self._task_tower_cfgs:
            mlp = config_to_kwargs(tc.mlp) if tc.HasField("mlp") else None
            for _ in range(self._task_domain_num if self._domain_input_name else 1):
                self._task_tower.append(TaskTower(self._task_input_dim, tc.num_class, mlp=mlp))

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        x = grouped[self._main_group_name]
        if self.epnet is not None:
            x = self.epnet(x, grouped[self._domain_group_name])
        task_inputs = self.ppnet(x, grouped[self._uia_group_name]) if self.ppnet is not None else [x]
        preds = {}
        D = self._task_domain_num
        for i, tc in enumerate(self._task_tower_cfgs):
            task_input = task_inputs[i] if self.ppnet is not None else task_inputs[0]
            if self._domain_input_name:
                for j in range(D):
                    preds.update(self._output_to_prediction(self._task_tower[i * D + j](task_input),
                                                            suffix=f"_{tc.tower_name}_{j}"))
            else:
                preds.update(self._output_to_prediction(self._task_tower[i](task_input), suffix=f"_{tc.tower_name}"))
        return preds

    def _select_domain_task_output(self, predictions: Dict[str, torch.Tensor], batch: Batch) -> Dict[str, torch.Tensor]:
        """pepnet.py:176-203 by comparison: `<name>` = sum_j [d == j] `<name>_<j>` for every per-domain prediction."""
        if not self._domain_input_name:
            return predictions
        d = batch.labels[self._domain_input_name]
        out = {}
        for tc in self._task_tower_cfgs:
            for kind in ("logits", "probs"):
                name = f"{kind}_{tc.tower_name}"
                sel = None
                for j in range(self._task_domain_num):
                    v = predictions[f"{name}_{j}"]
                    term = (d == j).to(v.dtype) * v
                    sel = term if sel is None else sel + term
                out[name] = sel
        return out

    def loss(self, predictions, batch):
        return super().loss(self._select_domain_task_output(predictions, batch), batch)

    def update_metric(self, predictions, batch, losses=None) -> None:
        super().update_metric(self._select_domain_task_output(predictions, batch), batch, losses)


class MultiTower(MultiTowerDIN):
    """tzrec/models/multi_tower.py:27-85: the same towers + final MLP without attention towers."""


class LinearCompressBlock(nn.Module):
    """tzrec/modules/interaction.py:236-264: W^T X with W [feature_num_in, feature_num_out]."""

    def __init__(self, feature_num_in: int, feature_num_out: int) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.empty((feature_num_in, feature_num_out)))
        nn.init.kaiming_uniform_(self.weight)

    def forward(self, inputs: torch.Tensor) -> torch.Tensor:
        return Fn.torch_linear_compress(inputs, self.weight)


class FactorizationMachineBlock(nn.Module):
    """tzrec/modules/interaction.py:267-321: LayerNorm(X (X^T W)) -> MLP -> Linear to feature_num_out x input_dim."""

    def __init__(self, input_dim: int, feature_num_in: int, feature_num_out: int, compressed_feature_num: int,
                 feature_num_mlp: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        self.feature_num_out, self.input_dim = feature_num_out, input_dim
        self.weight = nn.Parameter(torch.empty((feature_num_in, compressed_feature_num)))
        self.norm = nn.LayerNorm(feature_num_in * compressed_feature_num)
        self.mlp = MLP(in_features=feature_num_in * compressed_feature_num, **(feature_num_mlp or {}))
        self.feature_out_liner = _Linear(self.mlp.output_dim(), feature_num_out * input_dim)
        nn.init.kaiming_uniform_(self.weight)

    def forward(self, inputs: torch.Tensor) -> torch.Tensor:
        out = self.mlp(self.norm(Fn.torch_wukong_interaction(inputs, self.weight)))
        return self.feature_out_liner(out).view(-1, self.feature_num_out, self.input_dim)


class WuKongLayer(nn.Module):
    """tzrec/modules/interaction.py:324-378.  When Fn.wukong_usable holds, the FMB's interaction + norm, the LCB and the
    residual run as one kernel (Fn.wukong_mix), the FMB's MLP and output Linear on the dense path, and the residual
    add + LayerNorm(d) as a second kernel (Fn.wukong_out); otherwise the reference's torch formulation."""

    def __init__(self, input_dim: int, feature_num: int, lcb_feature_num: int, fmb_feature_num: int,
                 compressed_feature_num: int = 16, feature_num_mlp: Optional[Dict[str, Any]] = None) -> None:
        super().__init__()
        self.input_dim, self.feature_num = input_dim, feature_num
        self.lcb_feature_num, self.fmb_feature_num = lcb_feature_num, fmb_feature_num
        self.compressed_feature_num = compressed_feature_num
        self.lcb = LinearCompressBlock(feature_num, lcb_feature_num)
        self.fmb = FactorizationMachineBlock(input_dim, feature_num, fmb_feature_num, compressed_feature_num,
                                             feature_num_mlp)
        self.norm = nn.LayerNorm(input_dim)
        if feature_num != lcb_feature_num + fmb_feature_num:
            self.residual_projection = LinearCompressBlock(feature_num, lcb_feature_num + fmb_feature_num)
        else:
            self.residual_projection = nn.Identity()

    def output_feature_num(self) -> int:
        return self.lcb_feature_num + self.fmb_feature_num

    def fused_usable(self, inputs: torch.Tensor) -> bool:
        return Fn.wukong_usable(inputs, self.feature_num, self.input_dim, self.compressed_feature_num,
                                self.fmb_feature_num, self.lcb_feature_num)

    def forward(self, inputs: torch.Tensor) -> torch.Tensor:
        if self.fused_usable(inputs):
            f = self.fmb_feature_num
            w_res = None if isinstance(self.residual_projection, nn.Identity) else self.residual_projection.weight
            ln_f, base = Fn.wukong_mix(inputs, self.fmb.weight, self.fmb.norm.weight, self.fmb.norm.bias,
                                       self.lcb.weight, w_res, f)
            fmb_out = self.fmb.feature_out_liner(self.fmb.mlp(ln_f))
            return Fn.wukong_out(fmb_out, base, self.norm.weight, self.norm.bias, f)
        lcb = self.lcb(inputs)
        fmb = self.fmb(inputs)
        outputs = torch.concat((fmb, lcb), dim=1)
        return self.norm(outputs + self.residual_projection(inputs))


class WuKong(RankModel):
    """tzrec/models/wukong.py:26-130: the DLRM-style inputs (a `dense` group through a bottom MLP and a `sparse` group of
    equal-dim ids) through a stack of WuKong layers, then the final MLP and the output Linear."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        eg = self.embedding_group
        self._sparse_group_name = eg.group_names()[0] if len(eg.group_names()) == 1 else "sparse"
        self.dense_mlp = None
        self._dense_group_name = "dense"
        if len(eg.group_names()) > 1 and eg.has_group(self._dense_group_name):
            for name in eg.group_feature_dims(self._dense_group_name):
                if "seq_encoder" in name:
                    raise Exception("dense group not have sequence features.")
            self.dense_mlp = MLP(eg.group_total_dim(self._dense_group_name),
                                 **config_to_kwargs(self._model_config.dense_mlp))
        sparse_dims = eg.group_feature_dims(self._sparse_group_name)
        self._per_sparse_dim = 0
        for name, dim in sparse_dims.items():
            self._per_sparse_dim = dim
            if "seq_encoder" in name:
                raise Exception("sparse group not have sequence features.")
        self._sparse_num = len(sparse_dims)
        if len(set(sparse_dims.values())) > 1:
            raise Exception(f"sparse group feature dims must be the same, but we find {set(sparse_dims.values())}")
        if self.dense_mlp and self._per_sparse_dim != self.dense_mlp.output_dim():
            raise Exception("dense mlp last hidden_unit must be the same sparse feature dim")
        self._wukong_layers = nn.ModuleList()
        feature_num = self._sparse_num + (1 if self.dense_mlp else 0)
        for layer_cfg in self._model_config.wukong_layers:
            layer = WuKongLayer(self._per_sparse_dim, feature_num, **config_to_kwargs(layer_cfg))
            self._wukong_layers.append(layer)
            feature_num = layer.output_feature_num()
        self.final_mlp = MLP(feature_num * self._per_sparse_dim, **config_to_kwargs(self._model_config.final))
        self.output_mlp = _Linear(self.final_mlp.output_dim(), self._num_class)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        feat = grouped[self._sparse_group_name].reshape(-1, self._sparse_num, self._per_sparse_dim)
        if self.dense_mlp:
            dense_feat = self.dense_mlp(grouped[self._dense_group_name])
            feat = torch.cat([dense_feat.unsqueeze(1), feat], dim=1)
        for layer in self._wukong_layers:
            feat = layer(feat)
        y = self.output_mlp(self.final_mlp(feat.reshape(feat.size(0), -1)))
        return self._output_to_prediction(y)


def proto_float32(v: float) -> float:
    """A `float` proto field as MessageToDict hands it to config_to_kwargs (protobuf's ToShortestFloat): the fewest
    significant digits, from 6 up, that round-trip the stored float32 (0.3 stays 0.3, not 0.30000001192...)."""
    f32 = struct.unpack("f", struct.pack("f", float(v)))[0]
    precision = 6
    rounded = float(f"{f32:.{precision}g}")
    while struct.unpack("f", struct.pack("f", rounded))[0] != f32:
        precision += 1
        rounded = float(f"{f32:.{precision}g}")
    return rounded


class MaskBlock(nn.Module):
    """tzrec/modules/masknet.py:20-85: ffn(feature_input * mask_generator(mask_input)), with the reference's
    aggregation-width rule (reduction_ratio, when non-zero, overrides aggregation_dim) and its checks."""

    def __init__(self, input_dim: int, mask_input_dim: int, hidden_dim: int, reduction_ratio: float = 1.0,
                 aggregation_dim: int = 0) -> None:
        super().__init__()
        if not aggregation_dim and not reduction_ratio:
            raise ValueError("Either aggregation_dim or reduction_ratio must be provided.")
        if aggregation_dim:
            self.aggregation_dim = aggregation_dim
        if reduction_ratio:
            self.aggregation_dim = int(input_dim * reduction_ratio)
        assert self.aggregation_dim > 0, "aggregation_dim must be > 0, check your aggregation_dim or "
        self.mask_generator = nn.Sequential(_Linear(mask_input_dim, self.aggregation_dim), nn.ReLU(),
                                            _Linear(self.aggregation_dim, input_dim))
        assert hidden_dim > 0, "hidden_dim must be > 0."
        self._hidden_dim = hidden_dim
        self.ffn = nn.Sequential(_Linear(input_dim, hidden_dim), nn.LayerNorm(hidden_dim), nn.ReLU())

    def output_dim(self) -> int:
        return self._hidden_dim

    def fused_params(self):
        """(W1, b1, W2, b2, W3, b3, gamma, beta) in Fn.masknet_parallel's order."""
        g0, g2, f0, f1 = self.mask_generator[0], self.mask_generator[2], self.ffn[0], self.ffn[1]
        return (g0.weight, g0.bias, g2.weight, g2.bias, f0.weight, f0.bias, f1.weight, f1.bias)

    def forward(self, feature_input: torch.Tensor, mask_input: torch.Tensor) -> torch.Tensor:
        weights = self.mask_generator(mask_input)
        return self.ffn(feature_input * weights)


class MaskNetModule(nn.Module):
    """tzrec/modules/masknet.py:88-161.  In parallel mode, when Fn.masknet_usable holds, the blocks run as
    Fn.masknet_parallel: the mask generators' first layers as one GEMM, LN(e) * mask and the FFN's bias + LayerNorm +
    ReLU as fused kernels (csrc/tzk_masknet.cuh), every GEMM on 16-B aligned rows.  Serial mode, autocast, and shapes
    outside the kernels' cover take the reference's torch formulation."""

    def __init__(self, feature_dim: int, n_mask_blocks: int, mask_block: Dict[str, Any],
                 top_mlp: Optional[Dict[str, Any]] = None, use_parallel: bool = True, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        mask_block = dict(mask_block)
        if "reduction_ratio" in mask_block:
            mask_block["reduction_ratio"] = proto_float32(mask_block["reduction_ratio"])
        self.ln_emb = nn.LayerNorm(feature_dim)
        self.use_parallel = use_parallel
        if self.use_parallel:
            self.mask_blocks = nn.ModuleList([MaskBlock(feature_dim, feature_dim, **mask_block)
                                              for _ in range(n_mask_blocks)])
            self._output_dim = self.mask_blocks[0].output_dim() * n_mask_blocks
        else:
            self.mask_blocks = nn.ModuleList()
            self._output_dim = feature_dim
            for i in range(n_mask_blocks):
                self.mask_blocks.append(MaskBlock(self._output_dim, feature_dim, **mask_block))
                self._output_dim = self.mask_blocks[i].output_dim()
        self.top_mlp = None
        if top_mlp:
            self.top_mlp = MLP(in_features=self._output_dim, **top_mlp)
            self._output_dim = self.top_mlp.output_dim()

    def output_dim(self) -> int:
        return self._output_dim

    def fused_usable(self, feature_emb: torch.Tensor) -> bool:
        blk = self.mask_blocks[0] if len(self.mask_blocks) else None
        return blk is not None and Fn.masknet_usable(feature_emb, self.ln_emb.normalized_shape[0], blk.output_dim(),
                                                     len(self.mask_blocks), self.use_parallel)

    def forward(self, feature_emb: torch.Tensor) -> torch.Tensor:
        if self.fused_usable(feature_emb):
            hidden = Fn.masknet_parallel(feature_emb, self.ln_emb.weight, self.ln_emb.bias,
                                         [blk.fused_params() for blk in self.mask_blocks])
        else:
            ln_emb = self.ln_emb(feature_emb)
            if self.use_parallel:
                hidden = torch.concat([blk(ln_emb, feature_emb) for blk in self.mask_blocks], dim=-1)
            else:
                hidden = self.mask_blocks[0](ln_emb, feature_emb)
                for i in range(1, len(self.mask_blocks)):
                    hidden = self.mask_blocks[i](hidden, feature_emb)
        if self.top_mlp is not None:
            hidden = self.top_mlp(hidden)
        return hidden


class MaskNet(RankModel):
    """tzrec/models/masknet.py:25-71: the first feature group through MaskNetModule and a bias-less output Linear."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        feature_dim = self.embedding_group.group_total_dim(self.group_name)
        masknet_config = self._model_config.mask_net_module
        self.mask_net_layer = MaskNetModule(feature_dim, **config_to_kwargs(masknet_config))
        self.output_linear = _Linear(masknet_config.top_mlp.hidden_units[-1], self._num_class, bias=False)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        features = self.build_input(batch)[self.group_name]
        hidden = self.mask_net_layer(features)
        return self._output_to_prediction(self.output_linear(hidden))


class DBMTL(MultiTaskRank):
    """tzrec/models/dbmtl.py:28-175: the first feature group through an optional MaskNetModule, bottom MLP and MMoE,
    then per task tower its MLP, its relation MLP over [own net | relation towers' relation nets] in config order, and
    `task_outputs.i` (num_class outputs).  Towers take BCE or, on two-class heads, the JRC loss."""

    _TOWER_LOSSES = ("binary_cross_entropy", "jrc_loss")

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        if model_config.use_pareto_loss_weight:
            raise NotImplementedError("use_pareto_loss_weight is outside the hot-path scope")
        cfg = self._model_config
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        feature_in = self.embedding_group.group_total_dim(self.group_name)
        self.mask_net = None
        if cfg.HasField("mask_net"):
            self.mask_net = MaskNetModule(feature_in, **config_to_kwargs(cfg.mask_net))
            feature_in = self.mask_net.output_dim()
        self.bottom_mlp = None
        if cfg.HasField("bottom_mlp"):
            self.bottom_mlp = MLP(feature_in, **config_to_kwargs(cfg.bottom_mlp))
            feature_in = self.bottom_mlp.output_dim()
        self.mmoe = None
        if cfg.HasField("expert_mlp"):
            self.mmoe = MMoEModule(in_features=feature_in, expert_mlp=config_to_kwargs(cfg.expert_mlp),
                                   num_expert=cfg.num_expert, num_task=len(self._task_tower_cfgs),
                                   gate_mlp=config_to_kwargs(cfg.gate_mlp) if cfg.HasField("gate_mlp") else None)
            feature_in = self.mmoe.output_dim()
        self.task_mlps = nn.ModuleDict()
        for tc in self._task_tower_cfgs:
            if tc.HasField("mlp"):
                self.task_mlps[tc.tower_name] = MLP(feature_in, **config_to_kwargs(tc.mlp))
        self.relation_mlps = nn.ModuleDict()
        for tc in self._task_tower_cfgs:
            if tc.HasField("relation_mlp"):
                name = tc.tower_name
                dim = self.task_mlps[name].output_dim() if name in self.task_mlps else feature_in
                for rel in tc.relation_tower_names:
                    # dbmtl.py:98-108: a relation tower counts with its relation MLP, else its task MLP, else the
                    # tower input (whatever that tower's own output width is)
                    if rel in self.relation_mlps:
                        dim += self.relation_mlps[rel].output_dim()
                    elif rel in self.task_mlps:
                        dim += self.task_mlps[rel].output_dim()
                    else:
                        dim += feature_in
                self.relation_mlps[name] = MLP(dim, **config_to_kwargs(tc.relation_mlp))
        self.task_outputs = nn.ModuleList()
        for tc in self._task_tower_cfgs:
            name = tc.tower_name
            if name in self.relation_mlps:
                dim = self.relation_mlps[name].output_dim()
            elif name in self.task_mlps:
                dim = self.task_mlps[name].output_dim()
            else:
                dim = feature_in
            self.task_outputs.append(nn.Linear(dim, tc.num_class))

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        net = self.build_input(batch)[self.group_name]
        if self.mask_net is not None:
            net = self.mask_net(net)
        if self.bottom_mlp is not None:
            net = self.bottom_mlp(net)
        task_inputs = self.mmoe(net) if self.mmoe is not None else [net] * len(self._task_tower_cfgs)
        task_net = {}
        for i, tc in enumerate(self._task_tower_cfgs):
            name = tc.tower_name
            task_net[name] = self.task_mlps[name](task_inputs[i]) if name in self.task_mlps else task_inputs[i]
        relation_net = {}
        for tc in self._task_tower_cfgs:
            name = tc.tower_name
            if tc.HasField("relation_mlp"):
                x = torch.cat([task_net[name]] + [relation_net[r] for r in tc.relation_tower_names], dim=1)
                relation_net[name] = self.relation_mlps[name](x)
            else:
                relation_net[name] = task_net[name]
        return self._multi_task_output_to_prediction(
            [self.task_outputs[i](relation_net[tc.tower_name]) for i, tc in enumerate(self._task_tower_cfgs)])


class RocketLaunching(RankModel):
    """tzrec/models/rocket_launching.py:28-323: a booster MLP and a light MLP on the first feature group (after an
    optional share_mlp), each with its own output Linear.  The light net reads the shared input detached and is the one
    served; training adds the booster's loss, the hint MSE between the two heads' logits and, with
    feature_based_distillation, a similarity loss for every light hidden layer whose width matches a booster layer.

    Everything after the two MLPs (both Linears, the softmaxes and every loss) runs as one fused call each way when
    Fn.rocket_head_usable holds (csrc/tzk_rocket.cuh); predict stashes the losses for loss().  Otherwise the heads and
    losses are the reference's torch ops.  softmax_cross_entropy heads only; sample weights are refused."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        cfg = self._model_config
        kinds = [lc.WhichOneof("loss") for lc in model_config.losses]
        if not kinds or any(k != "softmax_cross_entropy" for k in kinds):
            raise NotImplementedError(f"RocketLaunching: losses {kinds} are outside the hot-path scope "
                                      "(softmax_cross_entropy only)")
        self.return_hidden_layer_feature = bool(cfg.feature_based_distillation)
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        feature_in = self.embedding_group.group_total_dim(self.group_name)
        self.share_mlp = None
        if cfg.HasField("share_mlp"):
            self.share_mlp = MLP(feature_in, **config_to_kwargs(cfg.share_mlp))
        in_dim = self.share_mlp.output_dim() if self.share_mlp else feature_in
        self.booster_mlp = MLP(in_dim, return_hidden_layer_feature=self.return_hidden_layer_feature,
                               **config_to_kwargs(cfg.booster_mlp))
        self.booster_linear = nn.Linear(self.booster_mlp.output_dim(), self._num_class)
        self.light_mlp = MLP(in_dim, return_hidden_layer_feature=self.return_hidden_layer_feature,
                             **config_to_kwargs(cfg.light_mlp))
        self.light_linear = nn.Linear(self.light_mlp.output_dim(), self._num_class)
        self.hint_loss_name = "hint_l2_loss"
        self.mlp_index_dict = self._get_distillation_mlp_index()
        sim = cfg.feature_distillation_function
        # any value but COSINE takes the reference's EUCLID branch (INNER_PRODUCT included)
        self._sim = Fn.ROCKET_COSINE if sim in ("COSINE", 0, "") else Fn.ROCKET_EUCLID
        self._head_losses = None

    def _get_distillation_mlp_index(self) -> Dict[int, int]:
        """light layer i -> the FIRST booster layer of the same width (several light layers may share one)."""
        booster = list(self._model_config.booster_mlp.hidden_units)
        out = {}
        for i, unit_i in enumerate(self._model_config.light_mlp.hidden_units):
            for j, unit_j in enumerate(booster):
                if unit_i == unit_j:
                    out[i] = j
                    break
        return out

    def _head_prediction(self, logits: torch.Tensor, probs: torch.Tensor, suffix: str) -> Dict[str, torch.Tensor]:
        preds = {"logits" + suffix: logits, "probs" + suffix: probs}
        if self._num_class == 2:
            preds["probs1" + suffix] = probs[:, 1]
        return preds

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        assert self._num_class > 1, "num_class must be greater than 1 when loss type is softmax_cross_entropy"
        net = self.build_input(batch)[self.group_name]
        share_net = self.share_mlp(net) if self.share_mlp is not None else net
        light_net = self.light_mlp(share_net.detach())
        light_h = light_net["hidden_layer_end"] if self.return_hidden_layer_feature else light_net
        booster_net = booster_h = None
        pairs = []
        if self.training:
            booster_net = self.booster_mlp(share_net)
            booster_h = booster_net["hidden_layer_end"] if self.return_hidden_layer_feature else booster_net
            if self.mlp_index_dict and not self.return_hidden_layer_feature:
                # the reference indexes the plain MLP outputs by layer name here and fails the same way
                raise TypeError("RocketLaunching: light and booster layers of equal width need "
                                "feature_based_distillation to expose their hidden layers")
            pairs = [(light_net[f"hidden_layer{i}"], booster_net[f"hidden_layer{j}"])
                     for i, j in self.mlp_index_dict.items()]
        hiddens = [light_h] + ([booster_h] if self.training else [])
        linears = [self.light_linear] + ([self.booster_linear] if self.training else [])
        fused_pairs = pairs if self.return_hidden_layer_feature else []
        self._head_losses = None
        if Fn.rocket_head_usable(hiddens, self._num_class, [l.shape[1] for l, _ in fused_pairs]):
            label = batch.labels.get(self._label_name) if self._label_name else None
            logits, probs, self._head_losses = Fn.rocket_head(
                [(h, m.weight, m.bias) for h, m in zip(hiddens, linears)], label, self._ce_smoothing, fused_pairs,
                self._sim)
        else:
            logits, probs, _ = Fn.torch_rocket_head(list(zip(hiddens, linears)), None)
        preds = self._head_prediction(logits[0], probs[0], "_light")
        if self.training:
            preds.update(self._head_prediction(logits[1], probs[1], "_booster"))
            for (i, j), (light, booster) in zip(self.mlp_index_dict.items(), pairs):
                preds[f"light_{i}"] = light
                preds[f"booster_{j}"] = booster
        return preds

    def loss(self, predictions: Dict[str, torch.Tensor], batch: Batch) -> Dict[str, torch.Tensor]:
        """rocket_launching.py:182-245: softmax_cross_entropy_booster (training), softmax_cross_entropy_light, then in
        training similarity_<i>_<j> per pair (feature_based_distillation) and hint_l2_loss."""
        losses, self._head_losses = self._head_losses, None
        distill = self.training and self.return_hidden_layer_feature
        if losses is None:
            logits = [predictions["logits_light"]] + ([predictions["logits_booster"]] if self.training else [])
            pairs = [(predictions[f"light_{i}"], predictions[f"booster_{j}"])
                     for i, j in self.mlp_index_dict.items()] if distill else []
            losses = Fn.torch_rocket_losses(logits, batch.labels[self._label_name], self._ce_smoothing, pairs,
                                            self._sim)
        ce_light, ce_booster, hint, *sims = losses
        out = {}
        if self.training:
            out["softmax_cross_entropy_booster"] = ce_booster
        out["softmax_cross_entropy_light"] = ce_light
        if self.training:
            if distill:
                for (i, j), s in zip(self.mlp_index_dict.items(), sims):
                    out[f"similarity_{i}_{j}"] = s
            out[self.hint_loss_name] = hint
        return out

    def _metric_heads(self):
        """rocket_launching.py:169-180: every metric and loss mean once per head, booster first."""
        m, l = list(self._base_model_config.metrics), list(self._base_model_config.losses)
        return [(m, l, self._label_name, "_booster"), (m, l, self._label_name, "_light")]

    def _updated_metric_heads(self):
        """rocket_launching.py:247-294: the booster head only in training; evaluation updates the light head alone."""
        heads = self._metric_heads()
        return heads if self.training else heads[1:]


class TDM(RankModel):
    """tzrec/models/tdm.py:28-105: the SEQUENCE group through MultiWindowDINEncoder, concatenated with the other
    groups in config order, then deep_mlp and output_mlp (num_class outputs; the example trains a two-class softmax
    cross-entropy head with auc on probs1).  The SEQUENCE group always hands its rows over jagged.  The tree sampler,
    tree construction and retrieval of the reference's TDM live in its data pipeline and are not part of the model."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        eg = self.embedding_group
        non_seq_fea_dim = 0
        self.seq_group_name = ""
        self.non_seq_group_name = []
        for fg in self._base_model_config.feature_groups:
            if eg.group_type(fg.group_name) == "SEQUENCE":
                self.seq_group_name = fg.group_name
            else:
                non_seq_fea_dim += eg.group_total_dim(fg.group_name)
                self.non_seq_group_name.append(fg.group_name)
        g = self.seq_group_name
        eg.set_jagged_for_attention([g])
        cfg = self._model_config.multiwindow_din
        self.multiwindow_din = MultiWindowDINEncoder(eg.group_total_dim(f"{g}.sequence"),
                                                     eg.group_total_dim(f"{g}.query"), g, list(cfg.windows_len),
                                                     config_to_kwargs(cfg.attn_mlp))
        self.deep_mlp = MLP(in_features=self.multiwindow_din.output_dim() + non_seq_fea_dim,
                            **config_to_kwargs(self._model_config.final))
        self.output_mlp = nn.Linear(self.deep_mlp.output_dim(), self._num_class)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        x = torch.cat([self.multiwindow_din(grouped)] + [grouped[n] for n in self.non_seq_group_name], dim=1)
        return self._output_to_prediction(self.output_mlp(self.deep_mlp(x)))


class CrossV2(nn.Module):
    """tzrec/modules/interaction.py:135-180: the low-rank cross network, x_{l+1} = x0 * v_l(u_l(x_l)) + x_l with
    u_kernels[l] = Linear(D, r, bias=False) and v_kernels[l] = Linear(r, D).  One fused call each way on the GPU
    (Fn.cross_v2) when Fn.cross_v2_usable holds; else the reference's loop (Fn.torch_cross_v2)."""

    def __init__(self, input_dim: int, cross_num: int = 3, low_rank: int = 32) -> None:
        super().__init__()
        self.cross_num = cross_num
        self._low_rank = low_rank
        self._input_dim = input_dim
        self.u_kernels = nn.ModuleList([nn.Linear(input_dim, low_rank, bias=False) for _ in range(cross_num)])
        self.v_kernels = nn.ModuleList([nn.Linear(low_rank, input_dim, bias=True) for _ in range(cross_num)])

    def output_dim(self) -> int:
        return self._input_dim

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        if Fn.cross_v2_usable(input, self.u_kernels, self.v_kernels):
            return Fn.cross_v2(input, self.u_kernels, self.v_kernels)
        return Fn.torch_cross_v2(input, self.u_kernels, self.v_kernels)


class DCNV2(RankModel):
    """tzrec/models/dcn_v2.py:26-88: the first feature group through an optional backbone MLP and the cross network,
    concatenated with an optional deep MLP on the raw group, then final and a bias-less output Linear."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        feature_dim = self.embedding_group.group_total_dim(self.group_name)
        cfg = self._model_config
        self.backbone = None
        if cfg.HasField("backbone"):
            self.backbone = MLP(in_features=feature_dim, **config_to_kwargs(cfg.backbone))
            feature_dim = self.backbone.output_dim()
        self.cross = CrossV2(input_dim=feature_dim, **config_to_kwargs(cfg.cross))
        final_input_dim = self.cross.output_dim()
        self.deep = None
        if cfg.HasField("deep"):
            self.deep = MLP(in_features=self.embedding_group.group_total_dim(self.group_name),
                            **config_to_kwargs(cfg.deep))
            final_input_dim += self.deep.output_dim()
        self.final = MLP(in_features=final_input_dim, **config_to_kwargs(cfg.final))
        self.output_mlp = nn.Linear(self.final.output_dim(), self._num_class, bias=False)

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        features = self.build_input(batch)[self.group_name]
        net = self.backbone(features) if self.backbone else features
        net = self.cross(net)
        if self.deep:
            net = torch.cat([net, self.deep(features)], dim=-1)
        return self._output_to_prediction(self.output_mlp(self.final(net)))


MODEL_CLASSES = {"dlrm": DLRM, "deepfm": DeepFM, "multi_tower_din": MultiTowerDIN, "multi_tower": MultiTower,
                 "mmoe": MMoE, "wukong": WuKong, "mask_net": MaskNet, "ple": PLE,
                 "pepnet": PEPNet, "dbmtl": DBMTL, "rocket_launching": RocketLaunching, "tdm": TDM,
                 "dcn_v2": DCNV2}


class JRCLoss(nn.Module):
    """tzrec/loss/jrc_loss.py:29-117: forward(logits [B, 2], labels [B], session_ids [B]) -> the [B] per-sample losses
    (reduction "none") or their mean ("mean", NaN for a batch without a positive or a negative, as the reference).  The
    mean runs tzk_jrc_loss on CUDA (functional.jrc_loss); "none" and CPU tensors take functional.torch_jrc_loss.  A
    label outside {0, 1} gives NaN where the reference raises."""

    def __init__(self, alpha: float = 0.5, reduction: str = "mean") -> None:
        super().__init__()
        if reduction not in ("mean", "none"):
            raise ValueError(f"reduction must be mean or none, got {reduction}")
        self._alpha, self._reduction = alpha, reduction

    def forward(self, logits: torch.Tensor, labels: torch.Tensor, session_ids: torch.Tensor) -> torch.Tensor:
        if self._reduction == "none":
            return Fn.torch_jrc_loss(logits, labels, session_ids, self._alpha, "none")
        return Fn.jrc_loss(logits, labels, session_ids, self._alpha)


def create_model(model_config: Message, features: List[BaseFeature], labels: List[str], device=None) -> RankModel:
    """tzrec/main.py:134-160 `_create_model` (class looked up from the `model` oneof)."""
    kind = model_config.WhichOneof("model")
    if kind not in MODEL_CLASSES:
        raise NotImplementedError(f"model {kind} is outside this repo's hot-path scope (supported: "
                                  f"{sorted(MODEL_CLASSES)})")
    return MODEL_CLASSES[kind](model_config, features, labels, device=device)


def sparse_optimizer_from_config(train_config: Message) -> SparseOptimizerSpec:
    """tzrec/optim/optimizer_builder.py:30-97 (sparse side)."""
    so = train_config.sparse_optimizer
    kind = so.WhichOneof("optimizer")
    cfg = getattr(so, kind)
    clip = dict(max_gradient=float(cfg.max_gradient) if cfg.gradient_clipping else 0.0)
    if kind == "sgd_optimizer":
        return SparseOptimizerSpec(kind=OPT_SGD, lr=cfg.lr, **clip)
    if kind == "adagrad_optimizer":
        return SparseOptimizerSpec(kind=OPT_ADAGRAD, lr=cfg.lr, initial_accumulator_value=cfg.initial_accumulator_value,
                                   **clip)
    if kind == "rowwise_adagrad_optimizer":
        modes = {"NONE": WD_NONE, "L2": WD_L2, "DECOUPLE": WD_DECOUPLE}
        mode = cfg.weight_decay_mode
        mode = modes[mode] if isinstance(mode, str) else int(mode)      # (an enum is its name, or its number)
        return SparseOptimizerSpec(kind=OPT_ROWWISE_ADAGRAD, lr=cfg.lr, weight_decay=cfg.weight_decay,
                                   weight_decay_mode=mode, **clip)
    adam_like = {"adam_optimizer": OPT_ADAM, "partial_rowwise_adam_optimizer": OPT_PARTIAL_ROWWISE_ADAM,
                 "lamb_optimizer": OPT_LAMB, "partial_rowwise_lamb_optimizer": OPT_PARTIAL_ROWWISE_LAMB}
    if kind in adam_like:
        return SparseOptimizerSpec(kind=adam_like[kind], lr=cfg.lr, beta1=cfg.beta1, beta2=cfg.beta2,
                                   weight_decay=cfg.weight_decay, **clip)
    if kind == "lars_sgd_optimizer":        # eta: fbgemm's default (the proto has no field for it)
        return SparseOptimizerSpec(kind=OPT_LARS_SGD, lr=cfg.lr, momentum=cfg.momentum, weight_decay=cfg.weight_decay,
                                   **clip)
    if kind in ("adadelta_optimizer", "rmsprop_optimizer"):
        # the reference raises the same way: the public torchrec / fbgemm-gpu releases have no such fused kernel
        raise RuntimeError(f"sparse {kind} is not available in the public torchrec / fbgemm-gpu releases (the "
                           "reference needs an unreleased fbgemm-gpu wheel for it), and is not implemented here")
    raise NotImplementedError(f"sparse optimizer {kind} is not implemented")


def dense_optimizer_from_config(train_config: Message, params, **kw) -> torch.optim.Optimizer:
    """tzrec/optim/optimizer_builder.py dense side: stock torch optimizers."""
    do = train_config.dense_optimizer
    kind = do.WhichOneof("optimizer")
    cfg = getattr(do, kind)
    if kind == "adam_optimizer":
        return torch.optim.Adam(params, lr=cfg.lr, betas=(cfg.beta1, cfg.beta2), weight_decay=cfg.weight_decay, **kw)
    if kind == "adamw_optimizer":
        return torch.optim.AdamW(params, lr=cfg.lr, betas=(cfg.beta1, cfg.beta2), weight_decay=cfg.weight_decay, **kw)
    if kind == "sgd_optimizer":
        return torch.optim.SGD(params, lr=cfg.lr, momentum=cfg.momentum, weight_decay=cfg.weight_decay)
    if kind == "adagrad_optimizer":
        return torch.optim.Adagrad(params, lr=cfg.lr, initial_accumulator_value=cfg.initial_accumulator_value)
    raise NotImplementedError(kind)


_MIXED_PRECISION_TO_DTYPE = {"BF16": torch.bfloat16, "FP16": torch.float16}


def mixed_precision_to_dtype(mixed_precision: Optional[str]) -> Optional[torch.dtype]:
    """train_config.mixed_precision -> autocast dtype (tzrec/acc/utils.py:267-286): empty means off, an unknown value
    raises."""
    if not mixed_precision:
        return None
    if mixed_precision not in _MIXED_PRECISION_TO_DTYPE:
        raise ValueError(f"Unknown mixed_precision: {mixed_precision}, "
                         f"available types: {list(_MIXED_PRECISION_TO_DTYPE.keys())}")
    return _MIXED_PRECISION_TO_DTYPE[mixed_precision]


class TrainWrapper(nn.Module):
    """tzrec/models/model.py:271-297: forward(batch) -> (total_loss, (losses, predictions, batch)), with `predict` and
    `loss` under torch.autocast(device type, mixed_dtype) when a mixed-precision dtype is given.

    The autocast weight-cast cache is off: a captured step (engine.GraphedTrainStep) then holds no cast tensor across
    replays, and the eager and the captured step run the same casts.  The cast values are the same either way; only a
    weight used twice in one forward is cast twice."""

    def __init__(self, model: RankModel, mixed_dtype: Optional[torch.dtype] = None, device_type: str = "cuda") -> None:
        super().__init__()
        self.model = model
        self.mixed_dtype, self.device_type = mixed_dtype, device_type

    def forward(self, batch: Batch):
        ctx = contextlib.nullcontext() if self.mixed_dtype is None else \
            torch.autocast(self.device_type, dtype=self.mixed_dtype, cache_enabled=False)
        with ctx:
            predictions = self.model.predict(batch)
            losses = self.model.loss(predictions, batch)
            total = torch.stack(list(losses.values())).sum()
        return total, (losses, {k: v.detach() for k, v in predictions.items()}, batch)
