"""Generates tests/golden/ref_dcn_v2.npz from the REFERENCE's own CrossV2, MLP and DCNV2 (run in the build container
only).

tzrec/modules/interaction.py CrossV2 and tzrec/models/dcn_v2.py DCNV2 run with their own code and the reference's
own MLP (tzrec/modules/mlp.py).  What DCNV2 imports from the rest of tzrec is stubbed: a RankModel whose
init_input / build_input hand over the seeded group features and whose prediction restates rank_model.py:133-160
(a one-logit sigmoid head, or softmax with probs1), and config_to_kwargs over plain dicts with the MLP defaults
filled in.

In float64, with state, inputs and upstream gradients rounded to float32 values first.  To keep the file small, those
(exact as float32) and the parameter gradients (rounded to float32 from the float64 result) are stored as float32;
outputs, input gradients, predictions and losses stay float64:
  mod_<case>:   CrossV2 alone (MODULE_CASES, (D, L, r)) with the reference's own initialisation after
                torch.manual_seed(0): state-dict keys and each entry's float64 sum (the state itself is redrawn by the
                tests from the same seed), the input, the output, the upstream gradient, and the gradients of the
                input and every parameter;
  model_<case>: DCNV2 (MODEL_CASES): keys, state, the group features, labels, predictions, the loss and the
                gradients of the group features and every parameter.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_dcn_v2_golden.py
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

# (D, L, r): the reference's module test CrossV2(32, 6, 2), its model test's cross (D 33, L 3, r 64), the docs
# example after its backbone, and D 256 at L 3
MODULE_CASES = {"d32_l6_r2": (32, 6, 2), "d33_l3_r64": (33, 3, 64), "d128_l2_r32": (128, 2, 32),
                "d256_l3_r32": (256, 3, 32)}
B_MODULE = 9
# the model cases: tzrec/models/dcn_v2_test.py's config (group of 33: no backbone, cross 3 x 64, deep [8, 4],
# final [2]), the same with a backbone, without deep, and two classes with softmax cross-entropy
MODEL_CASES = {
    "test_config": dict(D=33, backbone=None, cross=dict(cross_num=3, low_rank=64), deep=[8, 4], final=[2],
                        num_class=1),
    "backbone": dict(D=40, backbone=[24, 16], cross=dict(cross_num=2, low_rank=8), deep=[12], final=[8],
                     num_class=1),
    "no_deep": dict(D=24, backbone=None, cross=dict(cross_num=2, low_rank=4), deep=None, final=[8, 4],
                    num_class=1),
    "softmax2": dict(D=20, backbone=[16], cross=dict(cross_num=1, low_rank=6), deep=[8], final=[6], num_class=2),
}
B_MODEL = 12


class _Msg(dict):
    def __getattr__(self, k):
        v = self[k]
        return _Msg(v) if isinstance(v, dict) else v

    def HasField(self, k):
        return self.get(k) is not None


def _stub_model_packages(case, grouped):
    from torch import nn

    for name in ("tzrec.datasets", "tzrec.features"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    pb = types.ModuleType("tzrec.protos.model_pb2")
    pb.ModelConfig = object
    sys.modules[pb.__name__] = pb
    for name, attrs in {"tzrec.datasets.utils": {"Batch": object}, "tzrec.features.feature": {"BaseFeature": object}}.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    sys.modules["tzrec.utils.config_util"].config_to_kwargs = (
        lambda msg: dict(_MLP_DEFAULTS, **dict(msg)) if "hidden_units" in msg else dict(msg))

    class _Group:
        def group_names(self):
            return ["all"]

        def group_total_dim(self, name):
            return case["D"]

    class RankModel(nn.Module):
        def __init__(self, model_config, features, labels, sample_weights=None, **kwargs):
            super().__init__()
            self._model_config = model_config.dcn_v2
            self._num_class = model_config.num_class

        def init_input(self):
            self.embedding_group = _Group()

        def build_input(self, batch):
            return grouped

        def _output_to_prediction(self, output, suffix=""):
            if self._num_class == 1:
                output = torch.squeeze(output, dim=1)
                return {"logits": output, "probs": torch.sigmoid(output)}
            probs = torch.softmax(output, dim=1)
            return {"logits": output, "probs": probs, "probs1": probs[:, 1]}

    rm = types.ModuleType("tzrec.models.rank_model")
    rm.RankModel = RankModel
    sys.modules[rm.__name__] = rm


def _seeded_state(m, g):
    return {k: (torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.3).float().double()
            for k, v in m.state_dict().items()}


def main():
    _stub_packages()
    out = {}
    from tzrec.modules.interaction import CrossV2  # tzrec/modules/interaction.py:135

    for tag, (D, L, r) in MODULE_CASES.items():
        torch.manual_seed(0)
        mod = CrossV2(D, L, r).double()
        g = torch.Generator().manual_seed(D * 100 + L * 10 + r)
        sd = {k: v.float().double() for k, v in mod.state_dict().items()}      # the reference's own init
        mod.load_state_dict(sd)
        x = torch.randn(B_MODULE, D, generator=g, dtype=torch.float64).float().double().requires_grad_(True)
        y = mod(x)
        dy = torch.randn(y.shape, generator=g, dtype=torch.float64).float().double()
        y.backward(dy)
        pre = f"mod_{tag}_"
        out[pre + "shape"] = np.array([D, L, r])
        out[pre + "keys"] = np.array(list(mod.state_dict()))
        for k, v in sd.items():
            out[pre + "sdsum__" + k] = np.array(float(v.sum()))
        out[pre + "x"], out[pre + "dout"] = x.detach().float().numpy(), dy.float().numpy()
        out[pre + "out"], out[pre + "dx"] = y.detach().numpy(), x.grad.numpy()
        for k, p in mod.named_parameters():
            out[pre + "grad__" + k] = p.grad.float().numpy()

    for tag, case in MODEL_CASES.items():
        g = torch.Generator().manual_seed(len(tag))
        x = (torch.randn(B_MODEL, case["D"], generator=g, dtype=torch.float64) * 0.5).float().double()
        x.requires_grad_(True)
        grouped = {"all": x}
        _stub_model_packages(case, grouped)
        sys.modules.pop("tzrec.models.dcn_v2", None)
        from tzrec.models.dcn_v2 import DCNV2  # tzrec/models/dcn_v2.py:26

        cfg = {"cross": case["cross"], "final": {"hidden_units": case["final"]}}
        if case["backbone"]:
            cfg["backbone"] = {"hidden_units": case["backbone"]}
        if case["deep"]:
            cfg["deep"] = {"hidden_units": case["deep"]}
        torch.manual_seed(0)
        m = DCNV2(_Msg({"dcn_v2": cfg, "num_class": case["num_class"]}), [], ["clk"]).double()
        sd = _seeded_state(m, g)
        m.load_state_dict(sd)
        m.train()
        preds = m.predict(None)
        if case["num_class"] == 1:
            labels = torch.randint(0, 2, (B_MODEL,), generator=g).double()
            loss = torch.nn.BCEWithLogitsLoss(reduction="mean")(preds["logits"], labels)
        else:
            labels = torch.randint(0, case["num_class"], (B_MODEL,), generator=g)
            loss = torch.nn.CrossEntropyLoss(reduction="mean")(preds["logits"], labels)
        loss.backward()
        pre = f"model_{tag}_"
        out[pre + "keys"] = np.array(list(m.state_dict()))
        for k, v in sd.items():
            out[pre + "sd__" + k] = v.float().numpy()
        out[pre + "x"], out[pre + "dx"] = x.detach().float().numpy(), x.grad.numpy()
        out[pre + "labels"] = labels.numpy()
        for k, v in preds.items():
            out[pre + "pred__" + k] = v.detach().numpy()
        out[pre + "loss"] = np.array(loss.item())
        for k, p in m.named_parameters():
            out[pre + "grad__" + k] = p.grad.float().numpy()
    path = os.path.join(HERE, "ref_dcn_v2.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
