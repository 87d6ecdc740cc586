"""Generates tests/golden/ref_seq_encoders.npz from the REFERENCE's own SelfAttentionEncoder and PoolingEncoder (run
in the build container only).

tzrec/modules/sequence.py runs with its own code through the stub packages of make_golden_from_reference.py.  Each
module is built with the reference's own initialisation after torch.manual_seed(0) and run in float64.  To keep the file
small it stores each state entry's sum instead of the state: the tests rebuild the module from the same seed, and the
sums pin it.  Inputs are float32 values; outputs and gradients stay float64.

  sa_<case>:   SelfAttentionEncoder (SA_CASES): keys, state sums, padded sequence [B, T, D], lengths, output, upstream
               gradient; for cases whose every length equals T (after the crop) also the sequence's and every
               parameter's gradient.  Mixed-length cases store grads_nan: the reference's gradients there are NaN (its
               padded query rows see every key masked, and nan_to_num fixes only the forward).
  pool_<case>: PoolingEncoder (sum / mean, with and without a crop): padded sequence, lengths, output, d sequence.

    TZREC_REFERENCE=<checkout of alibaba/TorchEasyRec @ 54cac316> python tests/golden/make_seq_encoder_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_from_reference import _stub_packages  # noqa: E402

# name -> (D, E, H, max_len, lengths, T); lengths cover 0, 1 and beyond one 64-row key tile
SA_CASES = {
    "ref_test": (16, 32, 4, 0, [0, 1, 70, 5, 33], 75),      # the reference test's shape, T beyond the longest length
    "default": (48, 512, 8, 0, [3, 0, 1, 66, 20, 9], 66),
    "one_head": (8, 16, 1, 0, [4, 4, 4], 4),
    "hd_1": (8, 4, 4, 0, [5, 5, 5, 5], 5),
    "crop": (8, 16, 2, 3, [7, 3, 0, 5, 2, 9], 9),
    "equal": (16, 32, 4, 0, [6, 6, 6, 6], 6),
    "equal_crop": (8, 16, 2, 3, [5, 4, 3], 5),
}
# name -> (pooling_type, max_len)
POOL_CASES = {"sum": ("sum", 0), "mean": ("mean", 0), "sum_crop": ("sum", 3), "mean_crop": ("mean", 3)}
POOL_LENGTHS, POOL_D = [0, 1, 5, 2, 9, 4], 8


def _padded(g, lengths, T, D):
    seq = torch.zeros(len(lengths), T, D, dtype=torch.float64)
    for b, n in enumerate(lengths):
        seq[b, :n] = torch.randn(n, D, generator=g, dtype=torch.float64)
    return seq.float().double()


def main():
    _stub_packages()
    from tzrec.modules.sequence import PoolingEncoder, SelfAttentionEncoder  # tzrec/modules/sequence.py:174, 221

    out = {}
    for tag, (D, E, H, mx, lengths, T) in SA_CASES.items():
        torch.manual_seed(0)
        enc = SelfAttentionEncoder(D, "seq", E, num_heads=H, max_seq_length=mx).double()
        g = torch.Generator().manual_seed(len(tag))
        seq = _padded(g, lengths, T, D)
        lens = torch.tensor(lengths)
        dy = torch.randn(len(lengths), E, generator=g, dtype=torch.float64)
        st = seq.clone().requires_grad_(True)
        y = enc({"seq.sequence": st, "seq.sequence_length": lens})
        y.backward(dy)
        pre = f"sa_{tag}_"
        out[pre + "keys"] = np.array(list(enc.state_dict()))
        for k, v in enc.state_dict().items():
            out[pre + "sum__" + k] = np.array(float(v.sum()))
        out[pre + "shape"] = np.array([D, E, H, mx])
        out[pre + "seq"], out[pre + "lengths"] = seq.numpy(), np.array(lengths)
        out[pre + "out"], out[pre + "dout"] = y.detach().numpy(), dy.numpy()
        kept = [min(n, mx) if mx > 0 else n for n in lengths]
        equal = all(n == min(T, mx) if mx > 0 else n == T for n in kept)
        grads = [p.grad for _, p in enc.named_parameters()]
        out[pre + "grads_nan"] = np.array(any(bool(torch.isnan(t).any()) for t in grads))
        assert bool(out[pre + "grads_nan"]) == (not equal), tag
        if equal:
            out[pre + "dseq"] = st.grad.numpy()
            for k, p in enc.named_parameters():
                out[pre + "grad__" + k] = p.grad.numpy()

    g = torch.Generator().manual_seed(11)
    seq = _padded(g, POOL_LENGTHS, max(POOL_LENGTHS), POOL_D)
    dy = torch.randn(len(POOL_LENGTHS), POOL_D, generator=g, dtype=torch.float64)
    out["pool_seq"], out["pool_lengths"], out["pool_dout"] = seq.numpy(), np.array(POOL_LENGTHS), dy.numpy()
    for tag, (kind, mx) in POOL_CASES.items():
        enc = PoolingEncoder(POOL_D, "seq", pooling_type=kind, max_seq_length=mx)
        st = seq.clone().requires_grad_(True)
        y = enc({"seq.sequence": st, "seq.sequence_length": torch.tensor(POOL_LENGTHS)})
        y.backward(dy)
        out[f"pool_{tag}_out"], out[f"pool_{tag}_dseq"] = y.detach().numpy(), st.grad.numpy()

    path = os.path.join(HERE, "ref_seq_encoders.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
