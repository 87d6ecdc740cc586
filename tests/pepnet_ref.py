"""Float64 restatement of PEPNet's EPNet and PPNet (tzrec/modules/personalized_net.py), and of the fused gate product
stage on its own.

TEST INFRASTRUCTURE.  Written from the modules' definition: GateNU(g) = gamma * sigmoid(W2 ReLU(W1 g + b1) + b2);
EPNet(main, domain) = GateNU([domain | main.detach()]) * main; PPNet, per task i and depth j (module index
i * len_hidden + j): y_ij = act(Linear_ij(y_i,j-1)) * GateNU_ij([uia | main.detach()]), y_i,-1 = main (dropout 0 here).

`gate_fwd` / `gate_bwd` restate the fused kernels' stage (csrc/tzk_pepnet.cuh) in numpy float64, so each can be checked
alone; `run` composes the modules with torch float64 autograd for the golden fixture of the reference's own modules.
"""
import numpy as np
import torch

# tag: (B, main dim, domain dim or None (no EPNet), uia dim or None (no PPNet), epnet_hidden_unit or None (main dim),
#       tasks, ppnet hidden units, epnet gamma, ppnet gamma)
CASES = {
    # pepnet_taobao: group all 16 x 16 = 256, domain = occupation (16), uia 13 x 16 = 208, 2 tasks; its EPNet as is,
    # its PPNet with the hidden units 512-256 cut to 32-16 (the fixture stays small; the full widths are checked on
    # the GPU against the torch formulation)
    "taobao_ep": (3, 256, 16, None, None, 2, [], 2.0, 2.0),
    "taobao_pp": (3, 256, None, 208, None, 2, [32, 16], 2.0, 2.0),
    # tzrec/models/pepnet_test.py: group all 16 + 8 + 1 = 25, domain 16, uia 16, PPNet [16, 8] over 2 tasks; EPNet,
    # PPNet, and both
    "test_ep": (2, 25, 16, None, None, 2, [], 2.0, 2.0),
    "test_pp": (2, 25, None, 16, None, 2, [16, 8], 2.0, 2.0),
    "test_both": (2, 25, 16, 16, None, 2, [16, 8], 2.0, 2.0),
    # epnet_hidden_unit set (pepnet_test.py's second case sets 8), widths the fused path covers, both modules
    "hidden_set": (5, 24, 8, 16, 8, 3, [12, 8], 2.0, 2.0),
    # non-default gammas
    "gamma": (4, 20, 4, 12, 16, 2, [8, 4], 0.5, 1.5),
}


def sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def gate_fwd(segs):
    """segs [(x, bx or None, z, bz, relu, gamma)] -> [y] = act(x + bx) * gamma sigmoid(z + bz)."""
    out = []
    for x, bx, z, bz, relu, gamma in segs:
        a = x + (0.0 if bx is None else bx)
        h = np.maximum(a, 0.0) if relu else a
        out.append(h * (gamma * sigmoid(z + bz)))
    return out


def gate_bwd(segs, dys):
    """-> [(dx, dz, dbx, dbz)] of gate_fwd for the output gradients dys."""
    out = []
    for (x, bx, z, bz, relu, gamma), dy in zip(segs, dys):
        a = x + (0.0 if bx is None else bx)
        h = np.maximum(a, 0.0) if relu else a
        da = (a > 0).astype(np.float64) if relu else np.ones_like(a)
        s = sigmoid(z + bz)
        dx = dy * gamma * s * da
        dz = dy * h * gamma * s * (1 - s)
        out.append((dx, dz, dx.sum(0), dz.sum(0)))
    return out


def ordered_keys(tag):
    """The reference's state-dict keys of the case's modules (EPNet under `epnet.`, PPNet under `ppnet.`)."""
    B, M, Dd, U, eh, T, hidden, _, _ = CASES[tag]
    keys = []
    if Dd is not None:
        keys += [f"epnet.gate_nu.dense_layers.{i}.{p}" for i in (0, 2) for p in ("weight", "bias")]
    if U is not None:
        keys += [f"ppnet.linears.{k}.{p}" for k in range(T * len(hidden)) for p in ("weight", "bias")]
        keys += [f"ppnet.gate_nus.{k}.dense_layers.{i}.{p}" for k in range(T * len(hidden)) for i in (0, 2)
                 for p in ("weight", "bias")]
    return keys


def seeded_case(tag, seed=None):
    """(state dict with the reference's names, inputs {main, domain?, uia?}, dys [one per output]) of a case."""
    B, M, Dd, U, eh, T, hidden, _, _ = CASES[tag]
    rng = np.random.default_rng(sorted(CASES).index(tag) + 31 if seed is None else seed)
    sd = {}

    def lin(name, n_out, n_in):
        sd[name + ".weight"] = rng.uniform(-1, 1, (n_out, n_in)) / np.sqrt(n_in)
        sd[name + ".bias"] = rng.uniform(-1, 1, n_out) / np.sqrt(n_in)

    if Dd is not None:
        lin("epnet.gate_nu.dense_layers.0", eh or M, Dd + M)
        lin("epnet.gate_nu.dense_layers.2", M, eh or M)
    if U is not None:
        for i in range(T):
            n_in = M
            for j, h in enumerate(hidden):
                lin(f"ppnet.linears.{i * len(hidden) + j}", h, n_in)
                n_in = h
        for i in range(T):
            for j, h in enumerate(hidden):
                k = i * len(hidden) + j
                lin(f"ppnet.gate_nus.{k}.dense_layers.0", h, U + M)
                lin(f"ppnet.gate_nus.{k}.dense_layers.2", h, h)
    sd = {k: sd[k] for k in ordered_keys(tag)}
    inputs = {"main": rng.standard_normal((B, M))}
    if Dd is not None:
        inputs["domain"] = rng.standard_normal((B, Dd))
    if U is not None:
        inputs["uia"] = rng.standard_normal((B, U))
    n_out = T if U is not None else 1
    width = hidden[-1] if U is not None else M
    dys = [rng.standard_normal((B, width)) for _ in range(n_out)]
    return sd, inputs, dys


def run(tag, sd, inputs, dys):
    """float64 torch autograd of the restated modules -> (outputs, input gradients {name: grad}, parameter grads)."""
    B, M, Dd, U, eh, T, hidden, g_ep, g_pp = CASES[tag]
    P = {k: torch.tensor(v, requires_grad=True) for k, v in sd.items()}
    X = {k: torch.tensor(v, requires_grad=True) for k, v in inputs.items()}

    def gate_nu(pre, g, gamma):
        h = torch.relu(g @ P[pre + ".0.weight"].T + P[pre + ".0.bias"])
        return gamma * torch.sigmoid(h @ P[pre + ".2.weight"].T + P[pre + ".2.bias"])

    main = X["main"]
    if Dd is not None:
        main = gate_nu("epnet.gate_nu.dense_layers", torch.cat([X["domain"], main.detach()], 1), g_ep) * main
    if U is not None:
        g_in = torch.cat([X["uia"], main.detach()], 1)
        outs = []
        for i in range(T):
            y = main
            for j in range(len(hidden)):
                k = i * len(hidden) + j
                y = torch.relu(y @ P[f"ppnet.linears.{k}.weight"].T + P[f"ppnet.linears.{k}.bias"])
                y = y * gate_nu(f"ppnet.gate_nus.{k}.dense_layers", g_in, g_pp)
            outs.append(y)
    else:
        outs = [main]
    torch.autograd.backward(outs, [torch.tensor(d) for d in dys])
    return ([o.detach().numpy() for o in outs], {k: v.grad.numpy() for k, v in X.items()},
            {k: v.grad.numpy() for k, v in P.items()})
