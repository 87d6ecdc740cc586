"""Loader for tzrec pipeline configs (`examples/*.config`, protobuf text format) without protoc.

The reference compiles tzrec/protos/*.proto with grpc_tools (scripts/gen_proto.sh:23) and parses configs with
`text_format.Merge` (tzrec/utils/config_util.py:25-48).  Neither protoc nor the generated *_pb2 modules exist
here, so this module carries (a) a small text-format parser and (b) a hand-written schema for the messages the
hot path's five BASELINE configs touch (types, repeated-ness, defaults, oneofs — restated from
tzrec/protos/{pipeline,train,optimizer,data,feature,model,module,tower,models/*}.proto).  Fields or messages
outside the schema still parse generically (a field seen more than once, or written with [..], is repeated),
so every examples/*.config loads even when its model family is out of this repo's scope.

Like text_format.Merge, missing `required` fields are tolerated.  Enum values are plain strings
("DEEP", "WIDE", "FG_NONE", ...).
"""

import json
import re
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Tuple

# ---------------------------------------------------------------------------------------------------------
# schema: TYPE -> {field: (kind, repeated, default)}; kind in {"str","int","float","bool","enum"} or a TYPE name
# ---------------------------------------------------------------------------------------------------------
S, I, F, B, E = "str", "int", "float", "bool", "enum"


def _f(kind, default=None, rep=False):
    return (kind, rep, default)


_ID_FEATURE = {
    "feature_name": _f(S), "expression": _f(S), "embedding_name": _f(S), "embedding_dim": _f(I, 0),
    "hash_bucket_size": _f(I, 0), "num_buckets": _f(I, 0), "vocab_list": _f(S, rep=True), "value_dim": _f(I),
    "pooling": _f(S, "sum"), "default_value": _f(S, ""), "separator": _f(S, "\x1d"), "weighted": _f(B, False),
    "init_fn": _f(S), "use_mask": _f(B, False), "vocab_file": _f(S), "fg_encoded_default_value": _f(S),
    "default_bucketize_value": _f(I), "fg_value_type": _f(S), "trainable": _f(B, True), "stub_type": _f(B, False),
    "data_type": _f(S, "FP32"), "embedding_constraints": _f("ParameterConstraints"),
    "sequence_length": _f(I), "sequence_delim": _f(S, ";"), "sequence_fields": _f(S, rep=True),
    "zch": _f("ZeroCollisionHash"), "dynamicemb": _f("DynamicEmbedding"),
}
_RAW_FEATURE = {
    "feature_name": _f(S), "expression": _f(S), "embedding_name": _f(S), "embedding_dim": _f(I, 0),
    "boundaries": _f(F, rep=True), "value_dim": _f(I, 1), "normalizer": _f(S), "pooling": _f(S, "sum"),
    "default_value": _f(S, "0"), "separator": _f(S, "\x1d"), "init_fn": _f(S), "use_mask": _f(B, False),
    "fg_encoded_default_value": _f(S), "trainable": _f(B, True), "stub_type": _f(B, False),
    "data_type": _f(S, "FP32"), "embedding_constraints": _f("ParameterConstraints"),
    "sequence_length": _f(I), "sequence_delim": _f(S, ";"), "sequence_fields": _f(S, rep=True),
    "autodis": _f("AutoDisEmbedding"), "mlp": _f("MLPEmbedding"),
}
_LR_ONEOF = ["constant_learning_rate", "exponential_decay_learning_rate", "manual_step_learning_rate",
             "cosine_annealing_learning_rate", "cosine_annealing_warm_restarts_learning_rate"]
_FUSED = {"lr": _f(F, 0.002), "gradient_clipping": _f(B, False), "max_gradient": _f(F, 1.0)}
_FEATURE_KINDS = ["id_feature", "raw_feature", "combo_feature", "lookup_feature", "match_feature",
                  "sequence_feature", "expr_feature", "overlap_feature", "tokenize_feature", "custom_feature",
                  "kv_dot_product", "bool_mask_feature", "combine_feature", "sequence_id_feature",
                  "sequence_raw_feature", "sequence_combo_feature", "sequence_lookup_feature",
                  "sequence_match_feature", "sequence_expr_feature", "sequence_overlap_feature",
                  "sequence_tokenize_feature", "sequence_custom_feature", "sequence_kv_dot_product",
                  "sequence_bool_mask_feature", "sequence_combine_feature"]
_MODEL_KINDS = ["dlrm", "deepfm", "multi_tower", "multi_tower_din", "mask_net", "wide_and_deep", "dcn_v1",
                "dcn_v2", "xdeepfm", "wukong", "simple_multi_task", "mmoe", "dbmtl", "ple", "dc2vr", "dlrm_hstu",
                "pepnet", "ultra_hstu", "dssm", "dssm_v2", "dat", "hstu_match", "mind", "tdm", "rocket_launching",
                "sid_rqvae", "sid_rqkmeans"]

SCHEMA: Dict[str, Dict[str, Tuple[str, bool, Any]]] = {
    "EasyRecConfig": {
        "train_input_path": _f(S), "eval_input_path": _f(S), "model_dir": _f(S),
        "train_config": _f("TrainConfig"), "eval_config": _f("EvalConfig"), "export_config": _f("ExportConfig"),
        "data_config": _f("DataConfig"), "feature_configs": _f("FeatureConfig", rep=True),
        "model_config": _f("ModelConfig"),
    },
    "TrainConfig": {
        "sparse_optimizer": _f("SparseOptimizer"), "dense_optimizer": _f("DenseOptimizer"), "num_steps": _f(I),
        "num_epochs": _f(I), "save_checkpoints_steps": _f(I, 1000), "log_step_count_steps": _f(I, 100),
        "is_profiling": _f(B, False), "use_tensorboard": _f(B, True), "cudnn_allow_tf32": _f(B, True),
        "cuda_matmul_allow_tf32": _f(B, False), "global_embedding_constraints": _f("ParameterConstraints"),
        "mixed_precision": _f(S), "gradient_accumulation_steps": _f(I), "fine_tune_checkpoint": _f(S),
        "tensorboard_summaries": _f(S, rep=True), "grad_scaler": _f("GradScaler"),
    },
    "GradScaler": {"init_scale": _f(F, 65536.0), "growth_factor": _f(F, 2.0), "backoff_factor": _f(F, 0.5),
                   "growth_interval": _f(I, 2000)},
    "EvalConfig": {"num_steps": _f(I), "log_step_count_steps": _f(I, 100)},
    "SparseOptimizer": {
        "sgd_optimizer": _f("FusedSGDOptimizer"), "adagrad_optimizer": _f("FusedAdagradOptimizer"),
        "adam_optimizer": _f("FusedAdamOptimizer"), "rowwise_adagrad_optimizer": _f("FusedRowWiseAdagradOptimizer"),
        "partial_rowwise_adam_optimizer": _f("FusedAdamOptimizer"),     # same fields (optimizer.proto:124-131)
        "lars_sgd_optimizer": _f("FusedLarsSGDOptimizer"),
        "lamb_optimizer": _f("FusedAdamOptimizer"),                      # FusedLAMBOptimizer: the same fields
        "partial_rowwise_lamb_optimizer": _f("FusedAdamOptimizer"),      # FusedPartialRowWiseLAMBOptimizer: the same
        "adadelta_optimizer": _f("FusedAdadeltaOptimizer"), "rmsprop_optimizer": _f("FusedRMSpropOptimizer"),
        "constant_learning_rate": _f("ConstantLR"),
    },
    "DenseOptimizer": {
        "sgd_optimizer": _f("SGDOptimizer"), "adagrad_optimizer": _f("AdagradOptimizer"),
        "adam_optimizer": _f("AdamOptimizer"), "adamw_optimizer": _f("AdamWOptimizer"),
        "constant_learning_rate": _f("ConstantLR"), "part_optimizers": _f("PartOptimizer", rep=True),
    },
    "FusedSGDOptimizer": dict(_FUSED),
    "FusedAdagradOptimizer": dict(_FUSED, initial_accumulator_value=_f(F, 0.0)),
    "FusedRowWiseAdagradOptimizer": dict(_FUSED, weight_decay=_f(F, 0.0), weight_decay_mode=_f(E, "NONE")),
    "FusedAdamOptimizer": dict(_FUSED, beta1=_f(F, 0.9), beta2=_f(F, 0.999), weight_decay=_f(F, 0.0)),
    "FusedLarsSGDOptimizer": dict(_FUSED, momentum=_f(F, 0.9), weight_decay=_f(F, 0.0)),
    "FusedAdadeltaOptimizer": dict(_FUSED, rho=_f(F, 0.95), eps=_f(F, 1e-6), weight_decay=_f(F, 0.0)),
    "FusedRMSpropOptimizer": dict(_FUSED, alpha=_f(F, 0.99), eps=_f(F, 1e-8), weight_decay=_f(F, 0.0)),
    "SGDOptimizer": {"lr": _f(F, 0.002), "momentum": _f(F, 0.0), "dampening": _f(F, 0.0), "nesterov": _f(B, False),
                     "weight_decay": _f(F, 0.0)},
    "AdagradOptimizer": {"lr": _f(F, 0.002), "lr_decay": _f(F, 0.0), "weight_decay": _f(F, 0.0),
                         "initial_accumulator_value": _f(F, 0.0)},
    "AdamOptimizer": {"lr": _f(F, 0.002), "beta1": _f(F, 0.9), "beta2": _f(F, 0.999), "weight_decay": _f(F, 0.0)},
    "AdamWOptimizer": {"lr": _f(F, 0.002), "beta1": _f(F, 0.9), "beta2": _f(F, 0.999), "weight_decay": _f(F, 0.01)},
    "ConstantLR": {},
    "ParameterConstraints": {"sharding_types": _f(S, rep=True), "compute_kernels": _f(S, rep=True)},
    "DataConfig": {
        "batch_size": _f(I, 1024), "dataset_type": _f(E, "OdpsDataset"), "fg_mode": _f(E, "FG_NONE"),
        "label_fields": _f(S, rep=True), "num_workers": _f(I, 8), "odps_data_quota_name": _f(S, ""),
        "sample_weight_fields": _f(S, rep=True), "drop_remainder": _f(B, False), "fg_threads": _f(I, 1),
        "fg_encoded": _f(B), "input_fields": _f("Field", rep=True),
    },
    "FeatureConfig": {k: _f({"id_feature": "IdFeature", "raw_feature": "RawFeature",
                              "sequence_feature": "SequenceFeature", "sequence_id_feature": "IdFeature",
                              "sequence_raw_feature": "RawFeature"}.get(k, "Generic")) for k in _FEATURE_KINDS},
    "SeqFeatureConfig": {k: _f({"id_feature": "IdFeature", "raw_feature": "RawFeature"}.get(k, "Generic"))
                         for k in _FEATURE_KINDS if not k.startswith("sequence_")},
    "IdFeature": _ID_FEATURE,
    "RawFeature": _RAW_FEATURE,
    "SequenceFeature": {"sequence_name": _f(S), "sequence_length": _f(I), "sequence_delim": _f(S, ";"),
                        "sequence_pk": _f(S), "features": _f("SeqFeatureConfig", rep=True)},
    "ModelConfig": dict(
        {"feature_groups": _f("FeatureGroupConfig", rep=True), "num_class": _f(I, 1),
         "losses": _f("LossConfig", rep=True), "metrics": _f("MetricConfig", rep=True),
         "train_metrics": _f("TrainMetricConfig", rep=True), "kernel": _f(E, "PYTORCH"),
         "use_pareto_loss_weight": _f(B, False)},
        **{k: _f({"dlrm": "DLRM", "deepfm": "DeepFM", "mmoe": "MMoE", "multi_tower_din": "MultiTowerDIN",
                  "multi_tower": "MultiTower"}.get(k, "Generic")) for k in _MODEL_KINDS}),
    "FeatureGroupConfig": {"group_name": _f(S), "feature_names": _f(S, rep=True), "group_type": _f(E, "DEEP"),
                           "sequence_groups": _f("SeqGroupConfig", rep=True),
                           "sequence_encoders": _f("SeqEncoderConfig", rep=True),
                           "embedding_name_suffix": _f(S, "")},
    "SeqGroupConfig": {"group_name": _f(S), "feature_names": _f(S, rep=True), "embedding_name_suffix": _f(S, "")},
    "MLP": {"hidden_units": _f(I, rep=True), "dropout_ratio": _f(F, rep=True), "activation": _f(S, "nn.ReLU"),
            "use_bn": _f(B, False), "bias": _f(B, True), "use_ln": _f(B, False)},
    "DLRM": {"dense_mlp": _f("MLP"), "arch_with_sparse": _f(B, True), "final": _f("MLP")},
    "DeepFM": {"deep": _f("MLP"), "final": _f("MLP"), "wide_embedding_dim": _f(I, 4), "wide_init_fn": _f(S)},
    "MultiTower": {"towers": _f("Tower", rep=True), "final": _f("MLP")},
    "MultiTowerDIN": {"towers": _f("Tower", rep=True), "din_towers": _f("DINTower", rep=True), "final": _f("MLP")},
    "Tower": {"input": _f(S), "mlp": _f("MLP")},
    "DINTower": {"input": _f(S), "attn_mlp": _f("MLP")},
    "MMoE": {"expert_mlp": _f("MLP"), "gate_mlp": _f("MLP"), "num_expert": _f(I, 3),
             "task_towers": _f("TaskTower", rep=True)},
    "TaskTower": {"tower_name": _f(S), "label_name": _f(S), "metrics": _f("MetricConfig", rep=True),
                  "train_metrics": _f("TrainMetricConfig", rep=True), "losses": _f("LossConfig", rep=True),
                  "num_class": _f(I, 1), "mlp": _f("MLP"), "weight": _f(F, 1.0), "sample_weight_name": _f(S)},
    "LossConfig": {"binary_cross_entropy": _f("Generic"), "softmax_cross_entropy": _f("Generic"),
                   "l2_loss": _f("Generic"), "jrc_loss": _f("Generic"), "binary_focal_loss": _f("Generic")},
    "MetricConfig": {"auc": _f("AUC"), "multiclass_auc": _f("Generic"), "recall_at_k": _f("Generic"),
                     "mean_absolute_error": _f("Generic"), "mean_squared_error": _f("Generic"),
                     "accuracy": _f("Generic"), "grouped_auc": _f("Generic")},
    "AUC": {"thresholds": _f(I, 200)},
}

ONEOFS: Dict[str, Dict[str, List[str]]] = {
    "SparseOptimizer": {"optimizer": ["sgd_optimizer", "adagrad_optimizer", "adam_optimizer", "lars_sgd_optimizer",
                                      "lamb_optimizer", "partial_rowwise_lamb_optimizer",
                                      "partial_rowwise_adam_optimizer", "rowwise_adagrad_optimizer",
                                      "adadelta_optimizer", "rmsprop_optimizer"],
                        "learning_rate": _LR_ONEOF},
    "DenseOptimizer": {"optimizer": ["sgd_optimizer", "adagrad_optimizer", "adam_optimizer", "adamw_optimizer",
                                     "adadelta_optimizer", "rmsprop_optimizer"], "learning_rate": _LR_ONEOF},
    "FeatureConfig": {"feature": _FEATURE_KINDS},
    "SeqFeatureConfig": {"feature": [k for k in _FEATURE_KINDS if not k.startswith("sequence_")]},
    "ModelConfig": {"model": _MODEL_KINDS},
    "LossConfig": {"loss": ["binary_cross_entropy", "softmax_cross_entropy", "l2_loss", "jrc_loss",
                            "binary_focal_loss"]},
    "MetricConfig": {"metric": ["auc", "multiclass_auc", "recall_at_k", "mean_absolute_error",
                                "mean_squared_error", "accuracy", "grouped_auc"]},
    "RawFeature": {"dense_emb": ["autodis", "mlp"]},
}


class Message:
    """Tiny stand-in for a protobuf message (attribute access, HasField, WhichOneof, repeated fields as lists)."""

    def __init__(self, type_name: str = "Generic") -> None:
        object.__setattr__(self, "_type", type_name)
        object.__setattr__(self, "_values", OrderedDict())  # field -> list of raw values

    # ---- schema helpers -------------------------------------------------------------------------------
    def _spec(self, name: str) -> Optional[Tuple[str, bool, Any]]:
        return SCHEMA.get(self._type, {}).get(name)

    def _is_repeated(self, name: str) -> bool:
        spec = self._spec(name)
        if spec is not None:
            return spec[1]
        return len(self._values.get(name, [])) > 1 or name in getattr(self, "_bracketed", ())

    # ---- protobuf-like API ----------------------------------------------------------------------------
    def HasField(self, name: str) -> bool:
        return name in self._values and len(self._values[name]) > 0

    def WhichOneof(self, group: str) -> Optional[str]:
        found = None
        for f in ONEOFS.get(self._type, {}).get(group, []):
            if self.HasField(f):
                found = f
        return found

    def ListFields(self) -> List[Tuple[str, Any]]:
        return [(k, getattr(self, k)) for k in self._values]

    def CopyFrom(self, other: "Message") -> None:
        object.__setattr__(self, "_type", other._type)
        object.__setattr__(self, "_values", OrderedDict((k, list(v)) for k, v in other._values.items()))

    def __getattr__(self, name: str) -> Any:
        if name.startswith("_"):
            raise AttributeError(name)
        vals = self._values.get(name)
        spec = self._spec(name)
        if spec is None:
            if vals is None:
                if self._type in SCHEMA:
                    raise AttributeError(f"{self._type} has no field {name!r}")
                return None
            return vals if self._is_repeated(name) else vals[-1]
        kind, rep, default = spec
        if rep:
            if vals is None:
                vals = self._values.setdefault(name, [])
            return vals
        if vals:
            return vals[-1]
        if kind in (S, I, F, B, E):
            if default is not None:
                return default
            return {S: "", I: 0, F: 0.0, B: False, E: ""}[kind]
        return Message(kind)  # default (empty) sub-message, not attached

    def __setattr__(self, name: str, value: Any) -> None:
        spec = self._spec(name)
        if spec is not None and spec[1]:
            self._values[name] = list(value)
        else:
            self._values[name] = [value]

    def add(self, name: str) -> "Message":
        spec = self._spec(name)
        m = Message(spec[0] if spec else "Generic")
        self._values.setdefault(name, []).append(m)
        return m

    def to_dict(self) -> Dict[str, Any]:
        out = {}
        for k, vals in self._values.items():
            conv = [v.to_dict() if isinstance(v, Message) else v for v in vals]
            out[k] = conv if self._is_repeated(k) else conv[-1]
        return out

    def __repr__(self) -> str:
        return f"{self._type}({json.dumps(self.to_dict(), default=str)[:200]})"


# ---------------------------------------------------------------------------------------------------------
# text-format parser
# ---------------------------------------------------------------------------------------------------------
_TOKEN = re.compile(r"""
    (?P<ws>\s+|\#[^\n]*)
  | (?P<str>"(?:\\.|[^"\\])*"|'(?:\\.|[^'\\])*')
  | (?P<num>[-+]?(?:\d+\.?\d*(?:[eE][-+]?\d+)?|\.\d+(?:[eE][-+]?\d+)?)[fF]?)
  | (?P<id>[A-Za-z_][A-Za-z0-9_\.]*)
  | (?P<sym>[{}<>\[\]:,;])
""", re.X)

_ESC = {"n": "\n", "t": "\t", "r": "\r", "\\": "\\", '"': '"', "'": "'", "0": "\0"}


def _unescape(s: str) -> str:
    out, i = [], 0
    while i < len(s):
        c = s[i]
        if c == "\\" and i + 1 < len(s):
            n = s[i + 1]
            if n == "x":
                out.append(chr(int(s[i + 2:i + 4], 16)))
                i += 4
                continue
            if n.isdigit():
                j = i + 1
                while j < len(s) and j < i + 4 and s[j].isdigit():
                    j += 1
                out.append(chr(int(s[i + 1:j], 8)))
                i = j
                continue
            out.append(_ESC.get(n, n))
            i += 2
        else:
            out.append(c)
            i += 1
    return "".join(out)


def _tokenize(text: str) -> List[Tuple[str, str]]:
    toks, pos = [], 0
    while pos < len(text):
        m = _TOKEN.match(text, pos)
        if not m:
            line = text.count("\n", 0, pos) + 1
            raise ValueError(f"config parse error at line {line}: {text[pos:pos + 30]!r}")
        pos = m.end()
        kind = m.lastgroup
        if kind != "ws":
            toks.append((kind, m.group(kind)))
    return toks


class _Parser:
    def __init__(self, text: str) -> None:
        self.toks = _tokenize(text)
        self.i = 0

    def peek(self):
        return self.toks[self.i] if self.i < len(self.toks) else (None, None)

    def next(self):
        t = self.peek()
        self.i += 1
        return t

    def parse_message(self, msg: Message, closer: Optional[str]) -> Message:
        while True:
            kind, val = self.peek()
            if kind is None:
                if closer is not None:
                    raise ValueError("config parse error: unexpected end of input")
                return msg
            if kind == "sym" and val == closer:
                self.next()
                return msg
            if kind == "sym" and val in ",;":
                self.next()
                continue
            if kind != "id":
                raise ValueError(f"config parse error: expected a field name, got {val!r}")
            self.next()
            self.parse_field(msg, val)

    def parse_field(self, msg: Message, name: str) -> None:
        kind, val = self.peek()
        if kind == "sym" and val == ":":
            self.next()
            kind, val = self.peek()
        spec = msg._spec(name)
        if kind == "sym" and val in "{<":
            self.next()
            sub = Message(spec[0] if spec and spec[0] not in (S, I, F, B, E) else "Generic")
            self.parse_message(sub, "}" if val == "{" else ">")
            msg._values.setdefault(name, []).append(sub)
            return
        if kind == "sym" and val == "[":
            self.next()
            br = set(getattr(msg, "_bracketed", ()))
            br.add(name)
            object.__setattr__(msg, "_bracketed", br)
            msg._values.setdefault(name, [])
            while True:
                kind, val = self.peek()
                if kind == "sym" and val == "]":
                    self.next()
                    return
                if kind == "sym" and val == ",":
                    self.next()
                    continue
                if kind == "sym" and val in "{<":
                    self.next()
                    sub = Message(spec[0] if spec and spec[0] not in (S, I, F, B, E) else "Generic")
                    self.parse_message(sub, "}" if val == "{" else ">")
                    msg._values[name].append(sub)
                else:
                    msg._values[name].append(self.parse_scalar(spec))
        else:
            msg._values.setdefault(name, []).append(self.parse_scalar(spec))

    def parse_scalar(self, spec) -> Any:
        kind, val = self.next()
        want = spec[0] if spec else None
        if kind == "str":
            s = _unescape(val[1:-1])
            while self.peek()[0] == "str":  # adjacent string literals concatenate
                s += _unescape(self.next()[1][1:-1])
            return s
        if kind == "num":
            v = val.rstrip("fF")
            if want == F:
                return float(v)
            if want == I:
                return int(float(v))
            try:
                return int(v)
            except ValueError:
                return float(v)
        if kind == "id":
            if val in ("true", "True"):
                return True
            if val in ("false", "False"):
                return False
            if want == F and val in ("inf", "nan"):
                return float(val)
            return val  # enum identifier
        raise ValueError(f"config parse error: unexpected token {val!r}")


def parse_text(text: str, root_type: str = "EasyRecConfig") -> Message:
    return _Parser(text).parse_message(Message(root_type), None)


def load_pipeline_config(path: str) -> Message:
    """tzrec/utils/config_util.py:25-48: `.config` -> text format, `.json` -> JSON."""
    with open(path) as fh:
        text = fh.read()
    if path.endswith(".json"):
        return _from_dict(json.loads(text), "EasyRecConfig")
    return parse_text(text)


def _from_dict(d: Dict[str, Any], type_name: str) -> Message:
    msg = Message(type_name)
    for k, v in d.items():
        spec = msg._spec(k)
        sub_t = spec[0] if spec and spec[0] not in (S, I, F, B, E) else "Generic"
        vals = v if isinstance(v, list) else [v]
        msg._values[k] = [_from_dict(x, sub_t) if isinstance(x, dict) else x for x in vals]
    return msg


def config_to_kwargs(msg: Message) -> Dict[str, Any]:
    """tzrec/utils/config_util.py:68-72 (MessageToDict incl. default-valued fields, snake_case keys)."""
    out = {}
    for name, (kind, rep, default) in SCHEMA.get(msg._type, {}).items():
        v = getattr(msg, name)
        if isinstance(v, Message):
            if msg.HasField(name):
                out[name] = config_to_kwargs(v)
        elif rep:
            out[name] = [config_to_kwargs(x) if isinstance(x, Message) else x for x in v]
        else:
            out[name] = v
    for name in msg._values:
        if name not in out and msg._spec(name) is None:
            v = getattr(msg, name)
            out[name] = v.to_dict() if isinstance(v, Message) else v
    return out


def edit_config(msg: Message, edits: Dict[str, Any]) -> Message:
    """Dotted-path edits like tzrec/utils/config_util.py:182 (`a.b[0].c`), subset: attribute paths + [index]."""
    for path, value in edits.items():
        cur = msg
        parts = re.findall(r"([A-Za-z_][A-Za-z0-9_]*)(?:\[(\d+)\])?", path)
        for j, (name, idx) in enumerate(parts):
            last = j == len(parts) - 1
            if last and not idx:
                setattr(cur, name, value)
            else:
                nxt = getattr(cur, name)
                if idx:
                    if last:
                        nxt[int(idx)] = value
                        break
                    nxt = nxt[int(idx)]
                elif not cur.HasField(name):
                    cur._values[name] = [nxt]
                cur = nxt
    return msg
