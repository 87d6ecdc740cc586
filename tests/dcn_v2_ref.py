"""A float64 restatement of DCN-v2's cross network (tzrec/modules/interaction.py CrossV2.forward): the reference the
kernel tests compare against, and the tensors they feed it."""
import numpy as np
import torch


def cross_v2(x0: torch.Tensor, wu: torch.Tensor, wv: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """x_L for x0 [B, D], wu [L, r, D], wv [L, D, r], bias [L, D]: x_{l+1} = x0 * (V_l (U_l x_l) + c_l) + x_l."""
    x = x0
    for l in range(wu.shape[0]):
        x = x0 * ((x @ wu[l].T) @ wv[l].T + bias[l]) + x
    return x


def case(seed: int, B: int, D: int, L: int, r: int):
    """float64 (x0, wu, wv, bias) with nn.Linear's init scales, so the layers neither vanish nor blow up."""
    g = np.random.default_rng(seed)
    x0 = g.standard_normal((B, D))
    wu = g.uniform(-1, 1, (L, r, D)) / np.sqrt(D)
    wv = g.uniform(-1, 1, (L, D, r)) / np.sqrt(r)
    bias = g.uniform(-1, 1, (L, D)) / np.sqrt(r)
    return tuple(torch.from_numpy(t) for t in (x0, wu, wv, bias))


def grads(x0, wu, wv, bias, dy):
    """(y, dx0, d wu, d wv, d bias) of cross_v2 in float64."""
    leaves = [t.detach().clone().requires_grad_(True) for t in (x0, wu, wv, bias)]
    y = cross_v2(*leaves)
    y.backward(dy)
    return (y.detach(),) + tuple(t.grad for t in leaves)
