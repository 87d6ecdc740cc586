"""Float64 restatement of the JRC loss (tzrec/loss/jrc_loss.py) for the tests, and the seeded cases of
tests/golden/ref_dbmtl.npz.

TEST INFRASTRUCTURE.  `jrc` states the loss with explicit [B, B] session masks (small B only) and takes the gradient by
autograd in float64, independently of the O(B) formulations it checks (functional.torch_jrc_loss, csrc/tzk_jrc.cuh):

  ce_i = logsumexp(l0_i, l1_i) - l_{y_i, i}
  y_i = 1: ge_i = log(exp(l1_i) + sum_{j in s(i), y_j = 0} exp(l1_j)) - l1_i
  y_i = 0: ge_i = log(exp(l0_i) + sum_{j in s(i), y_j = 1} exp(l0_j)) - l0_i
  mean: mean_i(alpha ce_i + (1 - alpha) ge_i), NaN when the batch lacks a positive or a negative
  weighted: mean_i(w_i (alpha ce_i + (1 - alpha) ge_i))
"""
import numpy as np
import torch

ALPHAS = (0.5, 0.3)


def _layout(tag, B, rng):
    """(labels, session ids) of a golden layout."""
    if tag == "singletons":
        return (rng.random(B) < 0.3).astype(np.float64), rng.permutation(B).astype(np.int64) * 7 + 3
    if tag == "one_session":
        return (rng.random(B) < 0.3).astype(np.float64), np.full(B, 11, np.int64)
    if tag == "mixed":
        lens = [1, 2, 3, 5, 8, 13, 21, 34, 1, 1, 40]
        ids = np.concatenate([np.full(n, 1000 + 17 * k, np.int64) for k, n in enumerate(lens)])[:B]
        return (rng.random(B) < 0.4).astype(np.float64), rng.permutation(ids)
    if tag == "one_class_sessions":
        ids = rng.integers(0, 9, B).astype(np.int64)
        y = (ids % 3 == 0).astype(np.float64)                     # sessions 0, 3, 6 all positive, the rest negative
        y[ids == 4] = rng.random(int((ids == 4).sum())) < 0.5     # one session mixed
        return y, ids
    if tag in ("all_negative", "all_positive"):
        return np.full(B, 1.0 if tag == "all_positive" else 0.0), rng.integers(0, 5, B).astype(np.int64)
    if tag == "weighted":
        return (rng.random(B) < 0.35).astype(np.float64), rng.integers(0, 12, B).astype(np.int64)
    raise KeyError(tag)


# tag -> batch size
CASES = {"singletons": 37, "one_session": 61, "mixed": 128, "one_class_sessions": 90, "all_negative": 20,
         "all_positive": 9, "weighted": 77}


def seeded_case(tag):
    """(logits [B, 2], labels [B], session ids [B], weights [B] or None) in float64."""
    B = CASES[tag]
    rng = np.random.default_rng(sum(map(ord, tag)))
    logits = rng.normal(0.0, 2.0, (B, 2))
    y, s = _layout(tag, B, rng)
    w = rng.uniform(0.0, 2.0, B) if tag == "weighted" else None
    return logits, y, s, w


def jrc(logits, labels, sessions, alpha, weights=None):
    """-> (loss, d loss / d logits) in float64 numpy; weights None: the mean reduction."""
    with torch.enable_grad():
        return _jrc(logits, labels, sessions, alpha, weights)


def _jrc(logits, labels, sessions, alpha, weights):
    lg = torch.tensor(np.asarray(logits, np.float64), requires_grad=True)
    y = torch.tensor(np.asarray(labels, np.float64))
    s = torch.tensor(np.asarray(sessions, np.int64))
    B = y.shape[0]
    same = s[:, None] == s[None, :]
    eye = torch.eye(B, dtype=torch.bool)
    pos, neg = y == 1, y == 0
    ce = torch.logsumexp(lg, 1) - torch.where(pos, lg[:, 1], lg[:, 0])
    # row i's candidates: itself and the other class's samples of its session
    cand = eye | (same & torch.where(pos[:, None], neg[None, :], pos[None, :]))
    x = torch.where(pos[:, None], lg[:, 1][None, :].expand(B, B), lg[:, 0][None, :].expand(B, B))
    x = torch.where(cand, x, torch.full_like(x, float("-inf")))
    ge = torch.logsumexp(x, 1) - torch.where(pos, lg[:, 1], lg[:, 0])
    per = alpha * ce + (1 - alpha) * ge
    if weights is None:
        loss = per.mean()
        if not (bool(pos.any()) and bool(neg.any())):
            loss = loss + float("nan")
    else:
        loss = (per * torch.tensor(np.asarray(weights, np.float64))).mean()
    if B:
        loss.backward()
        grad = lg.grad.numpy()
    else:
        grad = np.zeros((0, 2))
    return float(loss.detach()), grad


# ---- DBMTL model cases (tzrec/models/dbmtl.py), as the dbmtl config's message tree -----------------------------------
MODEL_D, MODEL_B = 32, 16          # the group `all` width (two 16-wide id features) and the batch


def _mlp(*units):
    return {"hidden_units": list(units)}


def _tower(name, mlp=None, rel=(), rel_mlp=None, num_class=1):
    t = {"tower_name": name, "label_name": "clk", "num_class": num_class}
    if mlp:
        t["mlp"] = _mlp(*mlp)
    if rel:
        t["relation_tower_names"] = list(rel)
    if rel_mlp:
        t["relation_mlp"] = _mlp(*rel_mlp)
    return t


MODEL_CASES = {
    # dbmtl_taobao's shape, cut down; the cvr head two-class as in dbmtl_taobao_jrc
    "taobao": {"bottom_mlp": _mlp(24), "task_towers": [_tower("ctr", (16, 8)),
                                                       _tower("cvr", (16, 8), ("ctr",), (8,), num_class=2)]},
    "mask_net": {"mask_net": {"n_mask_blocks": 2, "mask_block": {"reduction_ratio": 2.0, "hidden_dim": 12},
                              "top_mlp": _mlp(16), "use_parallel": True},
                 "bottom_mlp": _mlp(12), "task_towers": [_tower("a", (8,)), _tower("b", (8,), ("a",), (4,))]},
    "mmoe": {"expert_mlp": _mlp(16, 12), "gate_mlp": _mlp(8), "num_expert": 3,
             "task_towers": [_tower("a", (8,)), _tower("b", (6,))]},
    "chain3": {"bottom_mlp": _mlp(20), "task_towers": [_tower("a", (8,)), _tower("b", (8,), ("a",), (6,)),
                                                      _tower("c", (4,), ("a", "b"), (5,))]},
    # a tower without an MLP, related to by another: its relation input counts with the tower input's width
    "no_mlp": {"bottom_mlp": _mlp(10), "task_towers": [_tower("a"), _tower("b", (6,), ("a",), (4,)),
                                                      _tower("c", None, ("b",), (3,))]},
}

_MLP_DEFAULTS = {"hidden_units": [], "dropout_ratio": [], "activation": "nn.ReLU", "use_bn": False, "bias": True,
                 "use_ln": False}


def model_kwargs(d):
    """config_to_kwargs of the case's sub-message: the proto defaults filled in, as MessageToDict with
    including_default_value_fields does (MLP and MaskNetModule / MaskBlock are the only nested kinds used)."""
    if "hidden_units" in d:
        return dict(_MLP_DEFAULTS, **d)
    if "n_mask_blocks" in d:
        out = {"use_parallel": True, **d}
        out["mask_block"] = {"reduction_ratio": 1.0, "aggregation_dim": 0, **d["mask_block"]}
        if "top_mlp" in d:
            out["top_mlp"] = model_kwargs(d["top_mlp"])
        return out
    return dict(d)


def model_config_text(tag):
    """The case as a pipeline config (two 16-wide id features in group `all`) for this repo's DBMTL."""
    def msg(d, ind):
        out = ""
        for k, v in d.items():
            if isinstance(v, dict):
                out += f"{ind}{k} {{\n{msg(v, ind + '    ')}{ind}}}\n"
            elif isinstance(v, list) and v and isinstance(v[0], dict):
                out += "".join(f"{ind}{k} {{\n{msg(x, ind + '    ')}{ind}}}\n" for x in v)
            elif isinstance(v, list):
                out += "".join(f'{ind}{k}: {x!r}\n'.replace("'", '"') for x in v)
            elif isinstance(v, bool):
                out += f"{ind}{k}: {'true' if v else 'false'}\n"
            else:
                out += f'{ind}{k}: {v!r}\n'.replace("'", '"')
        return out
    feats = "".join(f'feature_configs {{\n    id_feature {{\n        feature_name: "f{i}"\n        num_buckets: 50\n'
                    "        embedding_dim: 16\n    }\n}\n" for i in range(2))
    return ('data_config {\n    label_fields: "clk"\n}\n' + feats
            + 'model_config {\n    feature_groups {\n        group_name: "all"\n        feature_names: "f0"\n'
            '        feature_names: "f1"\n        group_type: DEEP\n    }\n    dbmtl {\n'
            + msg(MODEL_CASES[tag], "        ") + "    }\n}\n")


def seeded_state(tag, shapes):
    """Seeded parameters for the state-dict `shapes` {name: shape} (both sides load the same values), the input
    [B, D] and the output gradients {tower: [B, num_class]}."""
    rng = np.random.default_rng(sum(map(ord, "dbmtl_" + tag)))
    x = rng.normal(0.0, 1.0, (MODEL_B, MODEL_D))
    dys = {t["tower_name"]: rng.normal(0.0, 1.0, (MODEL_B, t["num_class"])) for t in MODEL_CASES[tag]["task_towers"]}
    sd = {k: rng.normal(0.0, 0.3, s) for k, s in shapes.items()}     # drawn last: x and dys do not depend on shapes
    return sd, x, dys
