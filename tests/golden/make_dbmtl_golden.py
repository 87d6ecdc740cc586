"""Generates tests/golden/ref_dbmtl.npz from the REFERENCE's own JRCLoss (run in the build container only).

tzrec/loss/jrc_loss.py is plain PyTorch: it is loaded through the stub parent packages of make_golden_from_reference.py
and run on the seeded layouts of tests/dbmtl_ref.py (`seeded_case`, which the tests call again), for alpha 0.5 and 0.3
and both reductions: "mean" in float64, "none" in float32 (its per-sample buffer is float32 whatever the input).  The mean reduction is the module's own; "none" is reduced as
rank_model.py:260-261 does, mean(loss * w), with w = 1 or the case's weights.  The fixture stores only what the
reference computes: the loss and d loss / d logits.

It also runs the reference's own DBMTL class on the model cases of tests/dbmtl_ref.py (MODEL_CASES: dbmtl_taobao's
shape cut down, with mask_net, with expert_mlp + gate_mlp, a relation chain of three towers, towers without an MLP).
dbmtl.py's own __init__ and predict run; what it imports from the rest of tzrec is stubbed (`_stub_model_packages`):
a MultiTaskRank whose embedding group is one group of the case's width and whose build_input hands over the seeded input,
plain-dict stand-ins for the generated protos, and config_to_kwargs over those dicts.  Stored: state-dict keys, the
seeded state, the towers' outputs, the input gradient and every parameter gradient, in float64.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_dbmtl_golden.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from dbmtl_ref import ALPHAS, CASES, MODEL_CASES, MODEL_D, model_kwargs, seeded_case, seeded_state  # noqa: E402
from make_golden_from_reference import REF, _stub_packages  # noqa: E402


def main():
    _stub_packages()
    loss_pkg = types.ModuleType("tzrec.loss")           # without its __init__, which imports every loss
    loss_pkg.__path__ = [os.path.join(REF, "tzrec", "loss")]
    sys.modules[loss_pkg.__name__] = loss_pkg
    from tzrec.loss.jrc_loss import JRCLoss  # tzrec/loss/jrc_loss.py:29

    out = {}
    for tag in CASES:
        logits, y, s, w = seeded_case(tag)
        for alpha in ALPHAS:
            for reduction in ("mean", "none"):
                if reduction == "mean" and w is not None:
                    continue
                # "none" builds its per-sample ge in a float32 buffer (jrc_loss.py:111), so it runs in float32
                dt = torch.float64 if reduction == "mean" else torch.float32
                lg = torch.tensor(logits, dtype=dt, requires_grad=True)
                loss = JRCLoss(alpha=alpha, reduction=reduction)(lg, torch.tensor(y).long(), torch.tensor(s))
                if reduction == "none":
                    loss = torch.mean(loss * (torch.tensor(w, dtype=dt) if w is not None else torch.ones(1, dtype=dt)))
                loss.backward()
                key = f"{tag}_{alpha}_{reduction}"
                out[key + "_loss"] = np.array(loss.item(), np.float64)
                out[key + "_dlogits"] = lg.grad.double().numpy()
    model_cases(out)
    path = os.path.join(HERE, "ref_dbmtl.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


class _Msg(dict):
    """A plain-dict stand-in for a generated proto message: attribute access and HasField."""

    def __getattr__(self, k):
        v = self[k] if k in self else {"num_expert": 3, "relation_tower_names": []}.get(k)
        if isinstance(v, dict):
            return _Msg(v)
        if isinstance(v, list):
            return [_Msg(x) if isinstance(x, dict) else x for x in v]
        return v

    def HasField(self, k):
        return k in self


def _stub_model_packages(group_dim):
    """What tzrec/models/dbmtl.py imports besides torch and its modules: Batch, BaseFeature, the generated protos,
    config_to_kwargs, and a MultiTaskRank whose embedding group has one group `all` of width group_dim, whose
    build_input returns the seeded input and whose _multi_task_output_to_prediction passes the towers' outputs on."""
    from torch import nn

    for name in ("tzrec.datasets", "tzrec.features", "tzrec.protos.models"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    mods = {}
    for name, attrs in {"tzrec.datasets.utils": {"Batch": object}, "tzrec.features.feature": {"BaseFeature": object},
                        "tzrec.protos.model_pb2": {"ModelConfig": object},
                        "tzrec.protos.models.multi_task_rank_pb2": {"DBMTL": _Msg}}.items():
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = mods[name] = m
    cu = sys.modules["tzrec.utils.config_util"]
    cu.config_to_kwargs = lambda msg: model_kwargs(dict(msg))

    class _EG:
        def group_names(self):
            return ["all"]

        def group_total_dim(self, name):
            return group_dim

    class MultiTaskRank(nn.Module):
        def __init__(self, model_config, features, labels, sample_weights=None, **kwargs):
            super().__init__()
            self._model_config = model_config.dbmtl

        def init_input(self):
            self.embedding_group = _EG()

        def build_input(self, batch):
            return {"all": batch}

        def _multi_task_output_to_prediction(self, outs):
            return outs

    mtr = types.ModuleType("tzrec.models.multi_task_rank")
    mtr.MultiTaskRank = MultiTaskRank
    sys.modules[mtr.__name__] = mtr


def model_cases(out):
    """The reference's own DBMTL (tzrec/models/dbmtl.py) on each MODEL_CASES tree: state-dict keys, the state it was
    run with, the towers' outputs, the input gradient and every parameter gradient."""
    _stub_model_packages(MODEL_D)
    from tzrec.models.dbmtl import DBMTL  # tzrec/models/dbmtl.py:28

    for tag, tree in MODEL_CASES.items():
        mc = _Msg({"dbmtl": tree})
        mc.WhichOneof = lambda group: "dbmtl"
        torch.manual_seed(0)
        m = DBMTL(mc, [], ["clk"]).double()
        sd, x, dys = seeded_state(tag, {k: tuple(v.shape) for k, v in m.state_dict().items()})
        m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
        xt = torch.from_numpy(x).requires_grad_(True)
        outs = m.predict(xt)
        torch.autograd.backward([outs[k] for k in dys], [torch.from_numpy(v) for v in dys.values()])
        out[f"model_{tag}_keys"] = np.array(list(m.state_dict()))
        for k, v in sd.items():
            out[f"model_{tag}_sd__{k}"] = v
        for k, v in outs.items():
            out[f"model_{tag}_out__{k}"] = v.detach().numpy()
        out[f"model_{tag}_dx"] = xt.grad.numpy()
        for k, p in m.named_parameters():
            out[f"model_{tag}_grad__{k}"] = p.grad.numpy()


if __name__ == "__main__":
    main()
