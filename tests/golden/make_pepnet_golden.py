"""Generates tests/golden/ref_pepnet.npz from the REFERENCE's own EPNet and PPNet (run in the build container only).

tzrec/modules/personalized_net.py is plain PyTorch: it is loaded file by file through the stub parent packages of
make_golden_from_reference.py, built with each case's shapes (EPNet under `epnet`, PPNet under `ppnet`, PPNet fed by
EPNet's output as tzrec/models/pepnet.py feeds it), and run on seeded parameters and inputs (tests/pepnet_ref.py
`seeded_case`, which the tests call again) with dropout 0.  The fixture stores only what the reference computes: outputs,
input gradients (main, domain, uia), every parameter gradient (rounded to float32 to keep the file small), and the
state-dict key list.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_pepnet_golden.py

Cases (tests/pepnet_ref.py CASES): pepnet_taobao's EPNet, and its PPNet with cut-down hidden units; the three module combinations of
tzrec/models/pepnet_test.py (group `all` 25 wide, PPNet [16, 8]); epnet_hidden_unit set; non-default gammas.
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
from pepnet_ref import CASES, seeded_case  # noqa: E402


def main():
    _stub_packages()
    from tzrec.modules.personalized_net import EPNet, PPNet  # tzrec/modules/personalized_net.py:62, :113

    out = {}
    for tag, (B, M, Dd, U, eh, T, hidden, g_ep, g_pp) in CASES.items():
        mods = nn.Module()
        mods.epnet = EPNet(M, Dd, hidden_dim=eh or M, gamma=g_ep) if Dd is not None else None
        mods.ppnet = PPNet(M, U, num_task=T, hidden_units=hidden, activation="nn.ReLU", dropout_ratio=[0.0],
                           gamma=g_pp) if U is not None else None
        sd, inputs, dys = seeded_case(tag)
        mods.double()
        mods.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
        xs = {k: torch.from_numpy(v).requires_grad_(True) for k, v in inputs.items()}
        x = xs["main"]
        if mods.epnet is not None:
            x = mods.epnet(x, xs["domain"])
        outs = mods.ppnet(x, xs["uia"]) if mods.ppnet is not None else [x]
        torch.autograd.backward(outs, [torch.from_numpy(d) for d in dys])
        out[f"{tag}_keys"] = np.array(list(mods.state_dict()))
        for i, o in enumerate(outs):
            out[f"{tag}_out{i}"] = o.detach().numpy()
        for k, v in xs.items():
            out[f"{tag}_d_{k}"] = v.grad.numpy()
        for name, p in mods.named_parameters():
            out[f"{tag}_grad__{name}"] = p.grad.numpy().astype(np.float32)
    path = os.path.join(HERE, "ref_pepnet.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
