"""Generates tests/golden/ref_rocket.npz from the REFERENCE's own RocketLaunching (run in the build container only).

tzrec/models/rocket_launching.py runs with its own __init__, predict, feature_based_sim, init_loss, _distillation_loss
and loss, and the reference's own MLP (tzrec/modules/mlp.py).  What it imports from the rest of tzrec is stubbed
(`_stub_model_packages`): a RankModel whose embedding group is one group `deep` of width D and whose build_input
hands over the seeded input, whose softmax_cross_entropy prediction, loss module and loss call restate
rank_model.py:147-155, 201-205 and 222-224; plain-dict stand-ins for the generated protos (Similarity: COSINE 0,
INNER_PRODUCT 1, EUCLID 2) and config_to_kwargs over those dicts with the MLP defaults filled in.

Per case of tests/rocket_ref.py (CASES), in float64 (state and input rounded to float32 values first): state-dict keys, the seeded state, input and labels, the training
predictions and every training loss, the input gradient and every parameter gradient of the sum of the losses, and
the eval predictions and losses.  The zero_light_row case sets every light_mlp bias to -1 and input row 0 to zero, so
row 0 of every light hidden layer is all zero.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_rocket_golden.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from rocket_ref import B, CASES, D, SIMILARITY  # noqa: E402
from make_golden_from_reference import _stub_packages  # noqa: E402

_MLP_DEFAULTS = dict(dropout_ratio=[], activation="nn.ReLU", use_bn=False, bias=True, use_ln=False)


class _Msg(dict):
    """A plain-dict stand-in for a generated proto message: attribute access and HasField (proto defaults of
    RocketLaunching for the fields a case leaves out)."""

    def __getattr__(self, k):
        v = self[k] if k in self else {"feature_based_distillation": False, "feature_distillation_function": 0}.get(k)
        return _Msg(v) if isinstance(v, dict) else v

    def HasField(self, k):
        return k in self


def _stub_model_packages():
    from torch import nn

    for name in ("tzrec.datasets", "tzrec.features"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    simi = types.ModuleType("tzrec.protos.simi_pb2")
    simi.Similarity = types.SimpleNamespace(**SIMILARITY)
    for name, attrs in {"tzrec.datasets.utils": {"Batch": object}, "tzrec.features.feature": {"BaseFeature": object},
                        "tzrec.protos.model_pb2": {"ModelConfig": object}}.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    sys.modules[simi.__name__] = simi
    cu = sys.modules["tzrec.utils.config_util"]
    cu.config_to_kwargs = lambda msg: dict(_MLP_DEFAULTS, **dict(msg))

    class _EG:
        def group_names(self):
            return ["deep"]

        def group_total_dim(self, name):
            return D

    class RankModel(nn.Module):
        def __init__(self, model_config, features, labels, sample_weights=None, **kwargs):
            super().__init__()
            self._base_model_config = model_config
            self._model_config = model_config.rocket_launching
            self._num_class = model_config.num_class
            self._label_name = labels[0]
            self._sample_weight_name = None
            self._loss_modules = {}
            self._loss_collection = {}

        def init_input(self):
            self.embedding_group = _EG()

        def build_input(self, batch):
            return {"deep": batch.x}

        def _output_to_prediction(self, output, suffix=""):
            probs = torch.softmax(output, dim=1)
            out = {"logits" + suffix: output, "probs" + suffix: probs}
            if self._num_class == 2:
                out["probs1" + suffix] = probs[:, 1]
            return out

        def _init_loss_impl(self, loss_cfg, num_class=1, reduction="none", suffix=""):
            self._loss_modules["softmax_cross_entropy" + suffix] = nn.CrossEntropyLoss(
                reduction=reduction, label_smoothing=loss_cfg.softmax_cross_entropy.label_smoothing)

        def _loss_impl(self, predictions, batch, label, loss_weight, loss_cfg, num_class=1, suffix=""):
            name = "softmax_cross_entropy" + suffix
            return {name: self._loss_modules[name](predictions["logits" + suffix], label)}

    rm = types.ModuleType("tzrec.models.rank_model")
    rm.RankModel = RankModel
    sys.modules[rm.__name__] = rm


def _tree(tag):
    sub, C, eps, _ = CASES[tag]
    rl = {}
    for k, v in sub.items():
        if k.endswith("_mlp"):
            rl[k] = {"hidden_units": v}
        elif k == "feature_distillation_function":
            rl[k] = SIMILARITY[v]
        else:
            rl[k] = v
    return _Msg({"rocket_launching": rl, "num_class": C,
                 "losses": [_Msg({"softmax_cross_entropy": {"label_smoothing": eps}})]})


def main():
    _stub_packages()
    _stub_model_packages()
    from tzrec.models.rocket_launching import RocketLaunching  # tzrec/models/rocket_launching.py:28

    out = {}
    for tag, (_, C, _, zero_row) in CASES.items():
        torch.manual_seed(0)
        m = RocketLaunching(_tree(tag), [], ["label"]).double()
        m.init_loss()
        g = torch.Generator().manual_seed(len(tag))
        sd = {k: torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.3 for k, v in m.state_dict().items()}
        x = torch.randn(B, D, generator=g, dtype=torch.float64)
        labels = torch.randint(0, C, (B,), generator=g)
        # values a float32 model holds exactly, so this repo's fp32 model runs on the very state and input
        sd = {k: v.float().double() for k, v in sd.items()}
        x = x.float().double()
        if zero_row:
            for k in sd:
                if k.startswith("light_mlp") and k.endswith("bias"):
                    sd[k].fill_(-1.0)
            x[0].zero_()
        m.load_state_dict(sd, strict=True)
        xt = x.clone().requires_grad_(True)
        batch = types.SimpleNamespace(x=xt, labels={"label": labels})
        m.train()
        preds = m.predict(batch)
        losses = m.loss(preds, batch)
        sum(losses.values()).backward()
        pre = f"{tag}_"
        out[pre + "keys"] = np.array(list(m.state_dict()))
        for k, v in sd.items():
            out[pre + "sd__" + k] = v.numpy()
        out[pre + "x"] = x.numpy()
        out[pre + "labels"] = labels.numpy()
        out[pre + "train_pred_keys"] = np.array(list(preds))
        for k, v in preds.items():
            out[pre + "train_pred__" + k] = v.detach().numpy()
        out[pre + "train_loss_keys"] = np.array(list(losses))
        for k, v in losses.items():
            out[pre + "train_loss__" + k] = np.array(v.item())
        out[pre + "dx"] = xt.grad.numpy()
        for k, p in m.named_parameters():
            out[pre + "grad__" + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).numpy()
        m.eval()
        with torch.no_grad():
            preds = m.predict(types.SimpleNamespace(x=x, labels={"label": labels}))
            losses = m.loss(preds, types.SimpleNamespace(x=x, labels={"label": labels}))
        out[pre + "eval_pred_keys"] = np.array(list(preds))
        for k, v in preds.items():
            out[pre + "eval_pred__" + k] = v.numpy()
        out[pre + "eval_loss_keys"] = np.array(list(losses))
        for k, v in losses.items():
            out[pre + "eval_loss__" + k] = np.array(v.item())
    path = os.path.join(HERE, "ref_rocket.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
