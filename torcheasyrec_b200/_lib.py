"""ctypes binding of libtzk.so — the C-ABI declared in include/tzk.h.

The library is the product: there is no CPU fallback.  `lib()` raises if the shared object is missing and
every wrapper in `kernels.py` raises if a tensor is not on a CUDA device.
"""

import ctypes
import os
from ctypes import c_char_p, c_float, c_int32, c_int64, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libtzk.so")

P = c_void_p  # every device pointer crosses the ABI as a plain address

class TzkOptArgs(ctypes.Structure):
    """struct tzk_opt_args (include/tzk.h)."""

    _fields_ = [("optimizer", c_int32), ("lr", c_float), ("eps", c_float), ("beta1", c_float), ("beta2", c_float),
                ("weight_decay", c_float), ("max_gradient", c_float), ("state", c_void_p), ("state2", c_void_p),
                ("step", c_void_p), ("weights_f16", c_int32), ("interleaved", c_int32), ("momentum", c_float),
                ("eta", c_float), ("weight_decay_mode", c_int32), ("per_sample_weights", c_void_p)]


# name -> (restype, argtypes); mirrors include/tzk.h one to one (tests/test_abi.py checks both directions)
SIGNATURES = {
    "tzk_abi_version": (c_int32, []),
    "tzk_last_error": (c_char_p, []),
    "tzk_sm_count": (c_int32, []),
    "tzk_lengths_to_offsets_workspace_bytes": (c_size_t, [c_int64]),
    "tzk_lengths_to_offsets": (c_int32, [P, c_int64, P, P, c_size_t, P]),
    "tzk_pooled_gather_fwd": (
        c_int32,
        [P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P],
    ),
    "tzk_seq_gather_fwd": (c_int32, [P, P, P, P, P, c_int32, c_int32, c_int32, c_int64, P, P]),
    "tzk_pooled_gather_fwd_f16": (
        c_int32,
        [P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P],
    ),
    "tzk_seq_gather_fwd_f16": (c_int32, [P, P, P, P, P, c_int32, c_int32, c_int32, c_int64, P, P]),
    "tzk_pooled_gather_fwd_strided": (
        c_int32,
        [P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P],
    ),
    "tzk_seq_gather_fwd_strided": (c_int32, [P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, c_int64, P, P]),
    "tzk_pooled_gather_fwd_weighted": (
        c_int32,
        [P, c_int32, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P],
    ),
    "tzk_fused_bwd_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int32]),
    "tzk_fused_bwd_weighted_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int32]),
    "tzk_fused_bwd_sort_weighted": (
        c_int32, [c_int32, P, P, P, P, P, c_int32, c_int32, c_int64, c_int64, c_int32, P, c_size_t, P]),
    "tzk_fused_bwd": (
        c_int32,
        [c_int32, c_int32, P, c_int64, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int64, c_int64, c_int32,
         c_int32, P, P, c_float, c_float, c_float, P, c_size_t, P],
    ),
    "tzk_fused_bwd_ex": (
        c_int32,
        [P, c_int32, P, c_int64, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int64, c_int64, c_int32, c_int32, P,
         c_float, P, c_size_t, P],
    ),
    "tzk_fused_bwd_apply_ex": (
        c_int32,
        [P, c_int32, P, c_int64, P, P, P, P, P, P, P, c_int32, c_int32, c_int64, c_int64, c_int32, c_int32, P,
         c_float, P, c_size_t, P],
    ),
    "tzk_fused_bwd_sort": (c_int32, [c_int32, P, P, P, P, c_int32, c_int32, c_int64, c_int64, c_int32, P, c_size_t, P]),
    "tzk_fused_bwd_apply": (
        c_int32,
        [c_int32, c_int32, P, c_int64, P, P, P, P, P, P, P, c_int32, c_int32, c_int64, c_int64, c_int32,
         c_int32, P, P, c_float, c_float, c_float, P, c_size_t, P],
    ),
    "tzk_bucketize_rw_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int32, c_int64]),
    "tzk_bucketize_rw": (
        c_int32,
        [P, P, c_int32, c_int32, c_int32, P, P, c_int64, c_int64, P, P, P, P, P, P, c_size_t, P],
    ),
    "tzk_bag_grad_expand": (c_int32, [P, c_int64, P, P, P, P, c_int32, c_int32, c_int32, P, P]),
    "tzk_permute_lengths": (c_int32, [P, P, c_int32, c_int32, P, P]),
    "tzk_permute_ids": (c_int32, [P, P, P, P, c_int32, c_int32, P, P]),
    "tzk_permute_weights": (c_int32, [P, P, P, P, c_int32, c_int32, P, P]),
    "tzk_col_gather_sum": (c_int32, [P, P, c_int32, P, P, P, c_int32, c_int64, P, c_int64, P]),
    "tzk_jagged_to_padded": (c_int32, [P, P, c_int32, c_int32, c_int32, P, P]),
    "tzk_padded_to_jagged": (c_int32, [P, P, c_int32, c_int32, c_int32, c_int64, P, P]),
    "tzk_fm_fwd": (c_int32, [P, c_int64, c_int64, c_int32, c_int32, P, c_int64, P]),
    "tzk_fm_bwd": (c_int32, [P, c_int64, P, c_int64, c_int64, c_int32, c_int32, P, c_int64, P]),
    "tzk_dot_interact_fwd": (
        c_int32,
        [P, c_int64, P, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, P, c_int64, P],
    ),
    "tzk_bias_act": (c_int32, [P, c_int64, P, c_int64, c_int32, c_int32, P]),
    "tzk_act_bwd_colsum_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "tzk_act_bwd_colsum": (c_int32, [P, c_int64, P, c_int64, c_int64, c_int32, c_int32, P, c_int64, P, P, c_size_t, P]),
    "tzk_small_linear_fwd": (c_int32, [P, c_int64, P, P, c_int64, c_int32, c_int32, c_int32, P, c_int64, P]),
    "tzk_small_linear_bwd_workspace_bytes": (c_size_t, [c_int64, c_int32, c_int32]),
    "tzk_small_linear_bwd": (
        c_int32,
        [P, c_int64, P, P, c_int64, P, c_int64, c_int64, c_int32, c_int32, c_int32, P, c_int64, P, P, P, c_size_t, P],
    ),
    "tzk_bce_logits_workspace_bytes": (c_size_t, [c_int64]),
    "tzk_bce_logits_fwd_bwd": (c_int32, [P, P, c_int64, P, P, P, c_size_t, P]),
    "tzk_dot_interact_bwd": (
        c_int32,
        [P, c_int64, P, c_int64, P, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, P, c_int64, P,
         c_int64, P],
    ),
    "tzk_interact_wide_bwd": (
        c_int32, [P, c_int64, P, c_int64, P, c_int64, P, c_int64, c_int64, P, c_int64, P, c_int64, P, P, P]),
    "tzk_tower_tail_bce_workspace_bytes": (c_size_t, [c_int64, c_int32, c_int32]),
    "tzk_tower_tail_bce": (c_int32, [P, c_int64, P, P, P, P, P, c_int64, c_int32, c_int32, P, P, c_int64, P, P, c_size_t, P]),
    "tzk_din_attn_input_fwd": (c_int32, [P, c_int64, c_int32, P, P, c_int32, c_int32, c_int64, P, P]),
    "tzk_din_attn_input_bwd": (c_int32, [P, P, c_int64, c_int32, P, P, c_int32, c_int32, c_int64, P, P, P]),
    "tzk_jagged_softmax_wsum_fwd": (c_int32, [P, P, P, c_int32, c_int32, c_int32, c_int64, P, P, P]),
    "tzk_jagged_softmax_wsum_bwd": (c_int32, [P, P, P, P, c_int32, c_int32, c_int32, c_int64, P, P, P]),
    "tzk_peer_pooled_gather_fwd": (
        c_int32, [P, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P, P, P]),
    "tzk_peer_pooled_gather_fwd_sel": (
        c_int32, [P, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P, P, P, c_int32, P]),
    "tzk_peer_seq_gather_fwd": (
        c_int32, [P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, c_int64, P, P, P, P]),
    "tzk_peer_mirror_refresh": (c_int32, [P, c_int32, P, P, P, P, c_int32, P, P]),
    "tzk_peer_barrier": (c_int32, [P, c_int32, c_int32, P, P]),
    "tzk_peer_bucketize_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int32]),
    "tzk_peer_bucketize": (
        c_int32, [P, P, c_int32, c_int32, c_int32, P, P, P, P, c_int32, c_int64, P, P, P, P, c_size_t, P]),
    "tzk_peer_publish_grad": (c_int32, [P, c_int64, P, P, P, P, c_int32, c_int32, P, c_int64, P]),
    "tzk_peer_push_grad": (
        c_int32, [P, P, c_int64, P, P, P, P, P, c_int32, c_int32, c_int64, c_int32, c_int32, c_int32, P]),
    "tzk_peer_allreduce_mean": (c_int32, [P, c_int32, c_int64, P, P]),
    "tzk_peer_small_update": (c_int32, [P, P, P, c_int32, P, c_int32, c_int32, c_int32, P, P]),
    "tzk_fused_bwd_sort_peer": (
        c_int32, [P, P, P, c_int32, c_int32, c_int64, c_int32, c_int64, c_int32, P, P, c_size_t, P]),
    "tzk_fused_bwd_apply_peer": (
        c_int32,
        [P, c_int32, P, c_int64, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, c_int64, c_int32, c_int64,
         c_int32, c_int32, P, c_float, P, c_size_t, P]),
    "tzk_peer_pooled_gather_fwd_weighted": (
        c_int32, [P, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P, P, P, P, c_int32, P]),
    "tzk_peer_bucketize_weighted": (
        c_int32, [P, P, c_int32, c_int32, c_int32, P, P, P, P, c_int32, c_int64, P, P, P, P, c_size_t, P, P, P]),
    "tzk_peer_push_grad_weighted": (
        c_int32, [P, P, c_int64, P, P, P, P, P, c_int32, c_int32, c_int64, c_int32, c_int32, c_int32, P, P]),
    "tzk_dot_interact27_fwd_bf16": (c_int32, [P, c_int64, P, c_int64, c_int64, P, c_int64, P]),
    "tzk_dot_interact27_bwd_bf16": (
        c_int32, [P, c_int64, P, c_int64, P, c_int64, c_int64, P, c_int64, P, c_int64, P]),
}

_lib = None


class TzkError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Loads libtzk.so (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise TzkError(
                f"{LIB_PATH} not found: build it with `python -m torcheasyrec_b200.csrc.build` "
                "(or __graft_entry__.build()).  There is no CPU fallback."
            )
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        if handle.tzk_abi_version() != 1:
            raise TzkError("libtzk ABI version mismatch; rebuild the library")
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().tzk_last_error()
        raise TzkError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
