"""Float64 restatement of PLE's extraction layers (tzrec/modules/extraction_net.py, stacked as tzrec/models/ple.py
stacks them), and of the fused gate stage on its own.

TEST INFRASTRUCTURE.  Written from the module's definition: per layer, `expert_num_per_task` MLP experts (Linear + ReLU
layers) per task on that task's input and `share_num` shared experts on the shared input; task gate i is a Linear with
bias over task i's input, softmax, mixing [task i experts..., shared experts...]; the shared gate (not in the last layer)
mixes [every task expert..., shared experts...] from the shared input.

`gates_fwd` / `gates_bwd` restate the fused kernels' stage (csrc/tzk_ple.cuh) in numpy float64, so each can be checked
alone; `stack` composes whole layers with torch float64 autograd for the golden fixture of the reference's own module.
"""
import numpy as np
import torch

# tag: (B, task input dims, shared input dim, one input tensor for all (PLE's first layer), layers, last layer final)
#   layer: (expert_num_per_task, share_num, task_expert_net units, share_expert_net units)
CASES = {
    # ple_taobao: 16 x 16 = 256 wide group, 2 tasks; each layer's gate widths (4 / 6, 6 / 9, 8) and final H
    # (256, 64, 32) with the expert hidden layers cut to 8 units
    "taobao": (3, [256, 256], 256, True, [(2, 2, [8, 256], [8, 256]), (3, 3, [8, 64], [8, 64]),
                                          (4, 4, [8, 32], [8, 32])], True),
    # tzrec/modules/extraction_net_test.py: task inputs 16 / 15 / 14, shared 13, final and not
    "extnet_final": (4, [16, 15, 14], 13, False, [(3, 4, [12, 8, 4], [12, 8, 6, 4])], True),
    "extnet": (4, [16, 15, 14], 13, False, [(3, 4, [12, 8, 4], [12, 8, 6, 4])], False),
    # tzrec/models/ple_test.py: group t1 = 16 + 8 + 1 = 25, 3 tasks, three layers
    "pletest": (2, [25, 25, 25], 25, True, [(3, 4, [12, 8, 4], [12, 8, 6, 4]), (3, 3, [8, 12, 8], [8, 12, 8]),
                                            (2, 2, [12, 6], [12, 6])], True),
    # share_num 0 in a layer that is not the last: the task gates mix their task's experts only, the shared gate every
    # task expert
    "share0": (5, [10, 10], 10, True, [(2, 0, [6, 5], [6, 5])], False),
}


def layer_dims(case):
    """[(task input dims, shared input dim, final)] per layer, by PLE's stacking rule."""
    _, in_dims, shared_dim, _, layers, last_final = case
    out = []
    for j, (_, _, tu, su) in enumerate(layers):
        final = last_final if j == len(layers) - 1 else False
        out.append((list(in_dims), shared_dim, final))
        in_dims, shared_dim = [tu[-1]] * len(in_dims), su[-1]
    return out


def seeded_case(tag, seed=None):
    """(state dict with the reference's names under `<layer>.`, inputs [task inputs..., shared input], dys) of a
    case; dys are the output gradients [task outputs..., shared output when the last layer is not final]."""
    case = CASES[tag]
    B, _, _, one_input, layers, _ = case
    rng = np.random.default_rng(sorted(CASES).index(tag) + 11 if seed is None else seed)
    sd = {}

    def lin(name, n_out, n_in):
        sd[name + ".weight"] = rng.uniform(-1, 1, (n_out, n_in)) / np.sqrt(n_in)
        sd[name + ".bias"] = rng.uniform(-1, 1, n_out) / np.sqrt(n_in)

    def mlp(prefix, n_in, units):
        for k, u in enumerate(units):
            lin(f"{prefix}.mlp.{k}.perceptron.0", u, n_in)
            n_in = u

    dims = layer_dims(case)
    for l, ((per, S, tu, su), (in_dims, shared_dim, final)) in enumerate(zip(layers, dims)):
        T = len(in_dims)
        for j in range(S):
            mlp(f"{l}._shared_layers.{j}", shared_dim, su)
        if not final:
            lin(f"{l}._shared_gate", T * per + S, shared_dim)
        for i, k in enumerate(in_dims):
            for j in range(per):
                mlp(f"{l}._task_layers.{i}.{j}", k, tu)
            lin(f"{l}._task_gates.{i}", per + S, k)
    sd = {k: v.astype(np.float32) for k, v in sd.items()}
    in_dims, shared_dim = dims[0][0], dims[0][1]
    if one_input:
        net = rng.standard_normal((B, shared_dim)).astype(np.float32)
        inputs = [net]
    else:
        inputs = [rng.standard_normal((B, k)).astype(np.float32) for k in in_dims + [shared_dim]]
    _, _, tu, su = layers[-1]
    n_out = len(in_dims) + (0 if dims[-1][2] else 1)
    dys = [rng.standard_normal((B, tu[-1] if i < len(in_dims) else su[-1])).astype(np.float32) for i in range(n_out)]
    return sd, inputs, dys


def ordered_keys(tag):
    """The state-dict key order of the reference's nn.ModuleList of ExtractionNets for a case."""
    case = CASES[tag]
    keys = []
    for l, ((per, S, tu, su), (in_dims, _, final)) in enumerate(zip(case[4], layer_dims(case))):
        for j in range(S):
            keys += [f"{l}._shared_layers.{j}.mlp.{k}.perceptron.0.{p}" for k in range(len(su)) for p in ("weight", "bias")]
        if not final:
            keys += [f"{l}._shared_gate.weight", f"{l}._shared_gate.bias"]
        for i in range(len(in_dims)):
            for j in range(per):
                keys += [f"{l}._task_layers.{i}.{j}.mlp.{k}.perceptron.0.{p}" for k in range(len(tu))
                         for p in ("weight", "bias")]
        for i in range(len(in_dims)):
            keys += [f"{l}._task_gates.{i}.weight", f"{l}._task_gates.{i}.bias"]
    return keys


def stack(tag, sd, inputs, dys):
    """-> (outputs, input gradients, {param name: gradient}) of the case's layers in float64 (torch autograd)."""
    case = CASES[tag]
    _, in_dims, _, one_input, layers, _ = case
    P = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in sd.items()}
    X = [torch.tensor(np.asarray(x, np.float64), requires_grad=True) for x in inputs]
    T = len(in_dims)
    task_in, shared_in = ([X[0]] * T, X[0]) if one_input else (X[:T], X[T])

    def mlp(prefix, x, n):
        for k in range(n):
            x = torch.relu(x @ P[f"{prefix}.mlp.{k}.perceptron.0.weight"].T + P[f"{prefix}.mlp.{k}.perceptron.0.bias"])
        return x

    def gate(name, x, experts):
        p = torch.softmax(x @ P[name + ".weight"].T + P[name + ".bias"], dim=1)
        return sum(p[:, e:e + 1] * ex for e, ex in enumerate(experts))

    shared_out = None
    for l, ((per, S, tu, su), (_, _, final)) in enumerate(zip(layers, layer_dims(case))):
        shared = [mlp(f"{l}._shared_layers.{j}", shared_in, len(su)) for j in range(S)]
        tasks = [[mlp(f"{l}._task_layers.{i}.{j}", task_in[i], len(tu)) for j in range(per)] for i in range(T)]
        outs = [gate(f"{l}._task_gates.{i}", task_in[i], tasks[i] + shared) for i in range(T)]
        shared_out = None if final else gate(f"{l}._shared_gate", shared_in, [e for t in tasks for e in t] + shared)
        task_in, shared_in = outs, shared_out
    outs = list(task_in) + ([] if shared_out is None else [shared_out])
    torch.autograd.backward(outs, [torch.tensor(np.asarray(d, np.float64)) for d in dys])
    return ([o.detach().numpy() for o in outs], [x.grad.numpy() for x in X],
            {k: v.grad.numpy() for k, v in P.items()})


# ---- the fused stage: one layer's gates -------------------------------------------------------------------------------
def _f64(a):
    return np.asarray(a, np.float64)


def gates_fwd(inputs, gate_input, weights, biases, experts, gate_experts):
    """-> y [n_gates, B, H], p [B, sum E_g] (the softmax of every gate, gate order)."""
    ys, ps = [], []
    for g, ids in enumerate(gate_experts):
        logit = _f64(inputs[gate_input[g]]) @ _f64(weights[g]).T + _f64(biases[g])
        e = np.exp(logit - logit.max(1, keepdims=True))
        p = e / e.sum(1, keepdims=True)
        ys.append(np.einsum("be,ebh->bh", p, np.stack([_f64(experts[x]) for x in ids])))
        ps.append(p)
    return np.stack(ys), np.concatenate(ps, 1)


def gates_bwd(inputs, gate_input, weights, biases, experts, gate_experts, dy):
    """dy [n_gates, B, H] -> (d_inputs per input, d_experts [n_experts, B, H], dW per gate, db per gate)."""
    _, p = gates_fwd(inputs, gate_input, weights, biases, experts, gate_experts)
    dy = _f64(dy)
    d_inputs = [np.zeros(_f64(x).shape) for x in inputs]
    d_experts = np.zeros((len(experts),) + _f64(experts[0]).shape)
    dW, db, o = [], [], 0
    for g, ids in enumerate(gate_experts):
        pg = p[:, o:o + len(ids)]
        o += len(ids)
        s = np.stack([(dy[g] * _f64(experts[x])).sum(1) for x in ids], 1)
        dl = pg * (s - (pg * s).sum(1, keepdims=True))
        for e, x in enumerate(ids):
            d_experts[x] += pg[:, e:e + 1] * dy[g]
        d_inputs[gate_input[g]] += dl @ _f64(weights[g])
        dW.append(dl.T @ _f64(inputs[gate_input[g]]))
        db.append(dl.sum(0))
    return d_inputs, d_experts, dW, db
