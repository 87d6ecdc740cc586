"""Model shells that consume the hot path: DLRM, DeepFM, MMoE, MultiTowerDIN (+ their dense blocks).

These are the callers of §8a rows A7-A10 (SURVEY.md §2 row 4): tzrec/models/{rank_model,dlrm,deepfm,mmoe,
multi_tower_din,multi_task_rank}.py and the dense blocks of tzrec/modules/{mlp,mmoe,sequence,task_tower}.py.
Dense towers stay plain PyTorch exactly as in the reference (parameter names are kept so state_dicts line up:
`dense_mlp.mlp.0.perceptron.0.weight`, ...).  The FM / dot-interaction steps are the tzk kernels.
"""

from typing import Any, Dict, List, Optional

import contextlib
import os

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
                 use_ln: bool = False, dim: int = 2, **_: Any) -> None:
        super().__init__()
        self.hidden_units = list(hidden_units)
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

    def forward(self, x: torch.Tensor, in_map=None) -> torch.Tensor:
        """`in_map`: column map of a zero-padded input (see dense_gemm.linear), consumed by the first layer."""
        for i, layer in enumerate(self.mlp):
            x = layer(x, in_map) if (i == 0 and in_map is not None) else layer(x)
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


# --------------------------------------------------------------------------------------------------------
# models
# --------------------------------------------------------------------------------------------------------
class RankModel(nn.Module):
    """tzrec/models/rank_model.py:40-287 reduced to: init_input / build_input / prediction dict / BCE loss."""

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
        for lc in model_config.losses:
            kind = lc.WhichOneof("loss")
            if kind not in (None, "binary_cross_entropy"):
                raise NotImplementedError(f"loss {kind} is outside the hot-path scope (BCE-with-logits only)")

    def init_input(self) -> None:
        """rank_model.py:83-112."""
        kw = {}
        if self._model_type == "deepfm":
            kw = dict(wide_embedding_dim=self._model_config.wide_embedding_dim or None,
                      wide_init_fn=self._model_config.wide_init_fn if self._model_config.HasField("wide_init_fn") else None)
        self.embedding_group = EmbeddingGroup(self._features, list(self._base_model_config.feature_groups),
                                              device=self._device, **kw)

    def build_input(self, batch: Batch) -> Dict[str, torch.Tensor]:
        """rank_model.py:114-131."""
        return self.embedding_group(batch)

    def _output_to_prediction(self, output: torch.Tensor, suffix: str = "") -> Dict[str, torch.Tensor]:
        """rank_model.py:133-179 for num_class == 1 binary heads."""
        assert self._num_class == 1, "only binary heads (num_class=1) are in scope"
        logits = torch.squeeze(output, dim=1)
        return {"logits" + suffix: logits, "probs" + suffix: torch.sigmoid(logits)}

    def loss(self, predictions: Dict[str, torch.Tensor], batch: Batch) -> Dict[str, torch.Tensor]:
        """rank_model.py:181-287: BCEWithLogitsLoss(mean) on the first label."""
        tail = getattr(self, "_tail_loss", None)
        if tail is not None:                 # computed together with the tower's tail (DLRM._fused_tail)
            self._tail_loss = None
            return {"binary_cross_entropy": tail}
        label = batch.labels[self._label_name].to(torch.float32)
        from .dense_gemm import bce_with_logits

        return {"binary_cross_entropy": bce_with_logits(predictions["logits"], label)}

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
        from .dense_gemm import InteractWideFn, _gemm3x_lib, interact_wide_usable

        first = self.final_mlp.mlp[0].perceptron
        if not (self._model_config.arch_with_sparse and len(first) == 2 and isinstance(first[1], nn.ReLU)
                and interact_wide_usable(dense_feat, sparse, first[0].weight, self._sparse_num, self._per_sparse_dim)):
            return None
        in_map = ((0, 0, 351), (351, 352, 432))
        return InteractWideFn.apply(_gemm3x_lib(), dense_feat, sparse, first[0].weight, first[0].bias, in_map)

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
        if (not self.training or Fn.autocast_dtype(all_feat) is not None or not torch.is_grad_enabled() or not all_feat.is_cuda or self._num_class != 1
                or not layers or self._label_name not in batch.labels or os.environ.get("TZK_FUSED_TAIL", "1") == "0"):
            return None
        last = layers[-1].perceptron
        if not (len(last) == 2 and isinstance(last[1], nn.ReLU)):     # Linear -> ReLU only (no BN / LN / dropout)
            return None
        label = batch.labels[self._label_name].to(torch.float32)
        w1, b1 = last[0].weight, last[0].bias
        w2, b2 = self.output_mlp.weight, self.output_mlp.bias
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


class MMoE(RankModel):
    """tzrec/models/mmoe.py:24-86 + multi_task_rank.py:50-65 (one BCE loss per tower, summed)."""

    def __init__(self, model_config, features, labels, sample_weights=None, **kwargs) -> None:
        super().__init__(model_config, features, labels, sample_weights, **kwargs)
        self._task_tower_cfgs = list(self._model_config.task_towers)
        self.init_input()
        self.group_name = self.embedding_group.group_names()[0]
        self.mmoe = MMoEModule(
            in_features=self.embedding_group.group_total_dim(self.group_name),
            expert_mlp=config_to_kwargs(self._model_config.expert_mlp), num_expert=self._model_config.num_expert,
            num_task=len(self._task_tower_cfgs),
            gate_mlp=config_to_kwargs(self._model_config.gate_mlp) if self._model_config.HasField("gate_mlp") else None)
        self._task_tower = nn.ModuleList()
        for cfg in self._task_tower_cfgs:
            # what the reference honours per tower (models/multi_task_rank.py:97-125) and this repo does not: refuse it
            # instead of silently training with plain mean BCE
            for fld in ("sample_weight_name", "task_space_indicator_label"):
                if cfg._spec(fld) is not None and cfg.HasField(fld) and getattr(cfg, fld):
                    raise NotImplementedError(f"task tower {cfg.tower_name}: {fld} is outside the hot-path scope")
            for lc in (cfg.losses if cfg._spec("losses") is not None else []):
                if lc.WhichOneof("loss") not in (None, "binary_cross_entropy"):
                    raise NotImplementedError(f"task tower {cfg.tower_name}: loss {lc.WhichOneof('loss')} is outside "
                                              "the hot-path scope (BCE-with-logits only)")
            mlp = config_to_kwargs(cfg.mlp) if cfg.HasField("mlp") else None
            self._task_tower.append(TaskTower(self.mmoe.output_dim(), cfg.num_class, mlp=mlp))

    def predict(self, batch: Batch) -> Dict[str, torch.Tensor]:
        grouped = self.build_input(batch)
        task_inputs = self.mmoe(grouped[self.group_name])
        preds = {}
        for i, cfg in enumerate(self._task_tower_cfgs):
            preds.update(self._output_to_prediction(self._task_tower[i](task_inputs[i]), suffix=f"_{cfg.tower_name}"))
        return preds

    def loss(self, predictions, batch):
        from .dense_gemm import bce_with_logits

        out = {}
        for cfg in self._task_tower_cfgs:
            label = batch.labels[cfg.label_name].to(torch.float32)
            out[f"binary_cross_entropy_{cfg.tower_name}"] = cfg.weight * bce_with_logits(
                predictions[f"logits_{cfg.tower_name}"], label)
        return out


class MultiTower(MultiTowerDIN):
    """tzrec/models/multi_tower.py:27-85: the same towers + final MLP without attention towers."""


MODEL_CLASSES = {"dlrm": DLRM, "deepfm": DeepFM, "multi_tower_din": MultiTowerDIN, "multi_tower": MultiTower,
                 "mmoe": MMoE}


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
