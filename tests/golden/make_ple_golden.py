"""Generates tests/golden/ref_ple.npz from the REFERENCE's own ExtractionNet (run in the build container only).

tzrec/modules/extraction_net.py is plain PyTorch: it is loaded file by file through the stub parent packages of
make_golden_from_reference.py, stacked as tzrec/models/ple.py stacks it (task input dims from output_dims[:-1], the
shared input dim from output_dims[-1], final_flag on the last layer) in an nn.ModuleList, and run on seeded parameters
and inputs (tests/ple_ref.py `seeded_case`, which the tests call again).  The fixture stores only what the reference
computes: outputs, input gradients, every parameter gradient, and the state-dict key list.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_ple_golden.py

Cases (tests/ple_ref.py CASES): ple_taobao's layer structure and gate widths with cut-down expert hidden layers; the
shapes of tzrec/modules/extraction_net_test.py, final and not; the three layers of tzrec/models/ple_test.py; a layer
stack with share_num 0.
"""
import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_from_reference import _stub_packages  # noqa: E402
from ple_ref import CASES, layer_dims, seeded_case  # noqa: E402


def main():
    _stub_packages()
    from tzrec.modules.extraction_net import ExtractionNet  # tzrec/modules/extraction_net.py:20

    out = {}
    for tag, case in CASES.items():
        _, in_dims, _, one_input, layers, _ = case
        nets = nn.ModuleList()
        for (per, S, tu, su), (ins, shared_dim, final) in zip(layers, layer_dims(case)):
            mlp = dict(activation="nn.ReLU", use_bn=False, dropout_ratio=0.0)
            nets.append(ExtractionNet(ins, shared_dim, network_name="layer", share_num=S, expert_num_per_task=per,
                                      share_expert_net=dict(hidden_units=su, **mlp),
                                      task_expert_net=dict(hidden_units=tu, **mlp), final_flag=final))
        sd, inputs, dys = seeded_case(tag)
        nets.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
        xs = [torch.from_numpy(x).requires_grad_(True) for x in inputs]
        T = len(in_dims)
        task_in, shared_in = ([xs[0]] * T, xs[0]) if one_input else (xs[:T], xs[T])
        for net in nets:
            task_in, shared_in = net(task_in, shared_in)
        outs = list(task_in) + ([] if shared_in is None else [shared_in])
        torch.autograd.backward(outs, [torch.from_numpy(d) for d in dys])
        out[f"{tag}_keys"] = np.array(list(nets.state_dict()))
        for i, o in enumerate(outs):
            out[f"{tag}_out{i}"] = o.detach().numpy()
        for i, x in enumerate(xs):
            out[f"{tag}_dx{i}"] = x.grad.numpy()
        for name, p in nets.named_parameters():
            out[f"{tag}_grad__{name}"] = p.grad.numpy()
    path = os.path.join(HERE, "ref_ple.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
