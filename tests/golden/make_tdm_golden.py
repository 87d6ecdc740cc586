"""Generates tests/golden/ref_tdm.npz from the REFERENCE's own MultiWindowDINEncoder and TDM (run in the build
container only).

tzrec/modules/sequence.py MultiWindowDINEncoder and tzrec/models/tdm.py TDM run with their own code and the
reference's own MLP (tzrec/modules/mlp.py).  What TDM imports from the rest of tzrec is stubbed: an EmbeddingGroup
whose group widths are the case's and whose forward hands over the seeded grouped features (the padded sequence
[B, T, C] with its lengths, the query and the DEEP groups), a RankModel whose softmax prediction restates
rank_model.py:147-155, model_pb2.SEQUENCE, and config_to_kwargs over plain dicts with the MLP defaults filled in.

In float64, with state and inputs rounded to float32 values first:
  enc_<case>: the encoder alone (ENC_CASES): state-dict keys and state, query, padded sequence, lengths, the output,
              the upstream gradient, and the gradients of query, sequence and every parameter;
  tdm_<key>:  the model (MODEL): keys, state, grouped inputs, labels, logits / probs / probs1, the softmax
              cross-entropy loss and the gradient of every parameter and input.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_tdm_golden.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_from_reference import _stub_packages  # noqa: E402

_MLP_DEFAULTS = dict(dropout_ratio=[], activation="nn.ReLU", use_bn=False, bias=True, use_ln=False)

# name -> (C, Dq, windows, attn hidden, activation, lengths); lengths cover 0, 1, exactly S and beyond S
ENC_CASES = {
    "example": (48, 48, [1, 1, 1, 2, 2, 2, 5, 6, 10, 20], [36], "nn.PReLU", [0, 1, 50, 63, 7, 19, 2, 33]),
    "w125_relu84": (16, 16, [1, 2, 5], [8, 4], "nn.ReLU", [0, 1, 8, 11, 3, 5, 2]),
    "relu842": (16, 16, [1, 2, 5], [8, 4, 2], "nn.ReLU", [4, 0, 1, 8, 9, 6]),
    "dq_lt_c": (16, 8, [2, 3], [8], "nn.PReLU", [0, 1, 5, 7, 3]),
}
# the model case: seq group C = 16 (Dq 16), DEEP groups user (16) and item (8); windows [1, 2, 5], attn [12] PReLU,
# final [16, 8] with BN, two classes
MODEL = dict(C=16, Dq=16, user=16, item=8, windows=[1, 2, 5], attn=[12], final=[16, 8],
             lengths=[0, 1, 8, 12, 3, 5, 2, 8, 6, 1])


class _Msg(dict):
    def __getattr__(self, k):
        v = self[k]
        return _Msg(v) if isinstance(v, dict) else v


def _stub_model_packages(grouped):
    from torch import nn

    for name in ("tzrec.datasets", "tzrec.features"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    pb = types.ModuleType("tzrec.protos.model_pb2")
    pb.SEQUENCE, pb.DEEP, pb.ModelConfig, pb.FeatureGroupConfig = "SEQUENCE", "DEEP", object, object
    for name, attrs in {"tzrec.datasets.utils": {"Batch": object}, "tzrec.features.feature": {"BaseFeature": object}}.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    sys.modules[pb.__name__] = pb
    sys.modules["tzrec.utils.config_util"].config_to_kwargs = lambda msg: dict(_MLP_DEFAULTS, **dict(msg))

    class EmbeddingGroup(nn.Module):
        def __init__(self, features, feature_groups):
            super().__init__()

        def group_total_dim(self, name):
            return {"seq.sequence": MODEL["C"], "seq.query": MODEL["Dq"], "user": MODEL["user"],
                    "item": MODEL["item"]}[name]

        def forward(self, batch):
            return grouped

    emb = types.ModuleType("tzrec.modules.embedding")
    emb.EmbeddingGroup = EmbeddingGroup
    sys.modules[emb.__name__] = emb

    class RankModel(nn.Module):
        def __init__(self, model_config, features, labels, sample_weights=None, **kwargs):
            super().__init__()
            self._model_config = model_config.tdm
            self._num_class = model_config.num_class

        def _output_to_prediction(self, output, suffix=""):
            probs = torch.softmax(output, dim=1)
            return {"logits": output, "probs": probs, "probs1": probs[:, 1]}

    rm = types.ModuleType("tzrec.models.rank_model")
    rm.RankModel = RankModel
    sys.modules[rm.__name__] = rm


def _padded(g, lengths, C):
    B, T = len(lengths), max(max(lengths), 1)
    seq = torch.zeros(B, T, C, dtype=torch.float64)
    for b, n in enumerate(lengths):
        seq[b, :n] = torch.randn(n, C, generator=g, dtype=torch.float64) * 0.5
    return seq.float().double()


def _seeded_state(m, g):
    sd = {}
    for k, v in m.state_dict().items():
        if not v.is_floating_point():
            sd[k] = v
        elif k.endswith("running_var"):
            sd[k] = (torch.rand(v.shape, generator=g, dtype=torch.float64) + 0.5).float().double()
        else:
            sd[k] = (torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.3).float().double()
    return sd


def main():
    _stub_packages()
    out = {}
    from tzrec.modules.sequence import MultiWindowDINEncoder  # tzrec/modules/sequence.py:288

    for tag, (C, Dq, windows, hidden, act, lengths) in ENC_CASES.items():
        torch.manual_seed(0)
        enc = MultiWindowDINEncoder(C, Dq, "seq", windows, dict(_MLP_DEFAULTS, hidden_units=hidden,
                                                                activation=act)).double()
        g = torch.Generator().manual_seed(len(tag))
        sd = _seeded_state(enc, g)
        enc.load_state_dict(sd)
        q = (torch.randn(len(lengths), Dq, generator=g, dtype=torch.float64) * 0.5).float().double()
        seq = _padded(g, lengths, C)
        lens = torch.tensor(lengths)
        dy = torch.randn(len(lengths), (len(windows) + 1) * C, generator=g, dtype=torch.float64)
        qt, st = q.clone().requires_grad_(True), seq.clone().requires_grad_(True)
        y = enc({"seq.query": qt, "seq.sequence": st, "seq.sequence_length": lens})
        y.backward(dy)
        pre = f"enc_{tag}_"
        out[pre + "keys"] = np.array(list(enc.state_dict()))
        for k, v in sd.items():
            out[pre + "sd__" + k] = v.numpy()
        out[pre + "windows"] = np.array(windows)
        out[pre + "hidden"] = np.array(hidden)
        out[pre + "act"] = np.array(act)
        out[pre + "query"], out[pre + "seq"], out[pre + "lengths"] = q.numpy(), seq.numpy(), np.array(lengths)
        out[pre + "out"], out[pre + "dout"] = y.detach().numpy(), dy.numpy()
        out[pre + "dquery"], out[pre + "dseq"] = qt.grad.numpy(), st.grad.numpy()
        for k, p in enc.named_parameters():
            out[pre + "grad__" + k] = p.grad.numpy()

    g = torch.Generator().manual_seed(7)
    lengths, B = MODEL["lengths"], len(MODEL["lengths"])
    grouped = {"seq.query": (torch.randn(B, MODEL["Dq"], generator=g, dtype=torch.float64) * 0.5).float().double(),
               "seq.sequence": _padded(g, lengths, MODEL["C"]), "seq.sequence_length": torch.tensor(lengths),
               "user": (torch.randn(B, MODEL["user"], generator=g, dtype=torch.float64) * 0.5).float().double(),
               "item": (torch.randn(B, MODEL["item"], generator=g, dtype=torch.float64) * 0.5).float().double()}
    for k in ("seq.query", "seq.sequence", "user", "item"):
        grouped[k].requires_grad_(True)
    _stub_model_packages(grouped)
    from tzrec.models.tdm import TDM  # tzrec/models/tdm.py:28

    cfg = _Msg({"feature_groups": [_Msg(group_name="seq", group_type="SEQUENCE"),
                                   _Msg(group_name="user", group_type="DEEP"),
                                   _Msg(group_name="item", group_type="DEEP")],
                "num_class": 2,
                "tdm": {"multiwindow_din": {"windows_len": MODEL["windows"],
                                            "attn_mlp": {"hidden_units": MODEL["attn"], "activation": "nn.PReLU"}},
                        "final": {"hidden_units": MODEL["final"], "use_bn": True}}})
    torch.manual_seed(0)
    m = TDM(cfg, [], ["clk"]).double()
    sd = _seeded_state(m, g)
    m.load_state_dict(sd)
    labels = torch.randint(0, 2, (B,), generator=g)
    m.train()
    preds = m.predict(None)
    loss = torch.nn.CrossEntropyLoss(reduction="mean")(preds["logits"], labels)
    loss.backward()
    out["tdm_keys"] = np.array(list(m.state_dict()))
    for k, v in sd.items():
        out["tdm_sd__" + k] = v.numpy()
    for k, v in grouped.items():
        out["tdm_in__" + k] = v.detach().numpy()
        if v.is_floating_point():
            out["tdm_din__" + k] = v.grad.numpy()
    out["tdm_labels"] = labels.numpy()
    for k, v in preds.items():
        out["tdm_pred__" + k] = v.detach().numpy()
    out["tdm_loss"] = np.array(loss.item())
    for k, p in m.named_parameters():
        out["tdm_grad__" + k] = p.grad.numpy()
    path = os.path.join(HERE, "ref_tdm.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
