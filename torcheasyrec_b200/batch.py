"""`Batch` — the hot path's input container — and a synthetic generator of it.

Layout contract = SURVEY.md §8a row A0 (tzrec/datasets/utils.py:299-342, built by DataParser.to_batch,
data_parser.py:402-594): `sparse_features[data_group]` is ONE KeyedJaggedTensor whose keys are the data
group's sparse feature names in config order (sequence features included, their lengths = sequence lengths),
`dense_features[data_group]` one KeyedTensor [B, sum value_dim], `labels[name]` [B].
`Batch` implements the Pipelineable protocol (`to`, `record_stream`, `pin_memory`; utils.py:344-463).
The reference's data IO (Arrow/ODPS readers, feature generation) is out of scope; benchmarks and tests feed
already-bucketised ids, exactly what DataParser emits in FG_NONE mode.
"""

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .features import BASE_DATA_GROUP, BaseFeature
from .sparse import JaggedTensor, KeyedJaggedTensor, KeyedTensor


@dataclass
class Batch:
    dense_features: Dict[str, KeyedTensor] = field(default_factory=dict)
    sparse_features: Dict[str, KeyedJaggedTensor] = field(default_factory=dict)
    sequence_mulval_lengths: Dict[str, KeyedJaggedTensor] = field(default_factory=dict)
    sequence_dense_features: Dict[str, JaggedTensor] = field(default_factory=dict)
    labels: Dict[str, torch.Tensor] = field(default_factory=dict)
    sample_weights: Dict[str, torch.Tensor] = field(default_factory=dict)
    tile_size: int = -1
    dummy: bool = False

    def _map(self, fn) -> "Batch":
        return Batch(
            dense_features={k: fn(v) for k, v in self.dense_features.items()},
            sparse_features={k: fn(v) for k, v in self.sparse_features.items()},
            sequence_mulval_lengths={k: fn(v) for k, v in self.sequence_mulval_lengths.items()},
            sequence_dense_features={k: fn(v) for k, v in self.sequence_dense_features.items()},
            labels={k: fn(v) for k, v in self.labels.items()},
            sample_weights={k: fn(v) for k, v in self.sample_weights.items()},
            tile_size=self.tile_size, dummy=self.dummy)

    def to(self, device, non_blocking: bool = False) -> "Batch":
        return self._map(lambda t: t.to(device, non_blocking=non_blocking))

    def pin_memory(self) -> "Batch":
        return self._map(lambda t: t.pin_memory())

    def record_stream(self, stream) -> None:
        for group in (self.dense_features, self.sparse_features, self.sequence_mulval_lengths, self.labels,
                      self.sample_weights):
            for v in group.values():
                if isinstance(v, torch.Tensor):
                    if v.is_cuda:
                        v.record_stream(stream)
                else:
                    v.record_stream(stream)

    def nbytes(self) -> int:
        """Bytes that cross PCIe when the batch is copied to the device."""
        n = 0
        for kjt in self.sparse_features.values():
            n += kjt.values().numel() * 8 + kjt.lengths().numel() * 4
        for kt in self.dense_features.values():
            n += kt.values().numel() * 4
        for t in self.labels.values():
            n += t.numel() * t.element_size()
        return n


def _draw_ids(rng: np.random.Generator, rows: int, n: int, dist: str) -> np.ndarray:
    if dist == "uniform" or rows <= 2:
        return rng.integers(0, rows, size=n, dtype=np.int64)
    if dist == "zipf":  # Zipf(s=1.05) clipped to the table (SURVEY.md §8d)
        return np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1).astype(np.int64)
    raise ValueError(dist)


def _behaviour_list(name: str, feats: Sequence[BaseFeature]) -> str:
    """The behaviour list a top-level sequence feature belongs to: `<list>__<field>` names (the reference's naming of a
    sequence group's fields, e.g. click_50_seq__adgroup_id) share `<list>` with every other top-level sequence feature
    of that prefix in the data group, so all of them get one length per sample; any other name is a list of its own."""
    head, sep, _ = name.partition("__")
    if not sep:
        return name
    peers = [f for f in feats
             if f.is_sparse and f.is_sequence and not f.sequence_name and f.name.startswith(head + "__")]
    return head + "__" if len(peers) > 1 else name


def synthetic_batch(features: Sequence[BaseFeature], batch_size: int, labels: Sequence[str], seed: int = 0,
                    id_dist: str = "uniform", seq_len_mix: bool = True,
                    label_cardinality: Optional[Dict[str, int]] = None) -> Batch:
    """Host (CPU) batch with the A0 layout for any id/raw/sequence feature list.

    Non-sequence id features get exactly one id per sample (Criteo / Taobao, L=1); grouped sequence features
    draw a length per sample from the mixture {0, 1, U[2,max], max} the reference's mock data uses
    (tzrec/tests/utils.py:157-182), one draw per behaviour list (_behaviour_list).  Labels are {0, 1} (1 with
    probability 0.25), except a label named in `label_cardinality`, which is drawn uniformly over [0, cardinality) (e.g. PEPNet's domain label)."""
    rng = np.random.default_rng(seed)
    B = batch_size
    by_group: Dict[str, List[BaseFeature]] = {}
    for f in features:
        by_group.setdefault(f.data_group, []).append(f)
    batch = Batch()
    seq_lengths: Dict[str, np.ndarray] = {}
    for dg, feats in by_group.items():
        keys, vals, lens, wts = [], [], [], []
        weighted = any(f.is_sparse and f.is_weighted for f in feats)
        dense_keys, dense_dims, dense_vals = [], [], []
        for f in feats:
            if f.is_sparse:
                if f.is_sequence:
                    sname = f.sequence_name or _behaviour_list(f.name, feats)
                    if sname not in seq_lengths:
                        mx = int(f.sequence_length or 50)
                        if seq_len_mix:
                            kind = rng.integers(0, 4, size=B)
                            L = np.where(kind == 0, 0, np.where(kind == 1, 1, np.where(
                                kind == 2, rng.integers(2, mx + 1, size=B), mx)))
                        else:
                            L = np.full(B, mx)
                        seq_lengths[sname] = L.astype(np.int32)
                    L = seq_lengths[sname]
                else:
                    L = np.ones(B, dtype=np.int32)
                keys.append(f.name)
                lens.append(L.astype(np.int32))
                vals.append(_draw_ids(rng, f.num_embeddings, int(L.sum()), id_dist))
                if weighted:      # as DataParser: weighted keys carry their weights, the others of the group 1.0
                    n = int(L.sum())
                    wts.append(rng.random(n, dtype=np.float32) if f.is_weighted else np.ones(n, dtype=np.float32))
            elif f.is_sequence:
                raise NotImplementedError("dense sequence features are not generated")
            else:
                dense_keys.append(f.name)
                dense_dims.append(f.value_dim)
                dense_vals.append(rng.random((B, f.value_dim), dtype=np.float32))
        if keys:
            batch.sparse_features[dg] = KeyedJaggedTensor(
                keys, torch.from_numpy(np.concatenate(vals)), lengths=torch.from_numpy(np.concatenate(lens)),
                weights=torch.from_numpy(np.concatenate(wts)) if weighted else None, stride=B)
        if dense_keys:
            batch.dense_features[dg] = KeyedTensor(dense_keys, dense_dims, torch.from_numpy(np.concatenate(dense_vals, axis=1)))
    for name in labels:
        if label_cardinality and name in label_cardinality:
            batch.labels[name] = torch.from_numpy(rng.integers(0, label_cardinality[name], size=B).astype(np.float32))
        else:
            batch.labels[name] = torch.from_numpy((rng.random(B) < 0.25).astype(np.float32))
    return batch
