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


PLE_MAX_GATES, PLE_MAX_EXPERTS, PLE_MAX_GATE_EXPERTS = 9, 64, 32


class TzkPleGateArgs(ctypes.Structure):
    """struct tzk_ple_gate_args (include/tzk.h): one PLE extraction layer's gates."""

    _fields_ = [("B", c_int64), ("H", c_int32), ("n_experts", c_int32), ("n_inputs", c_int32), ("n_gates", c_int32),
                ("in_dim", c_int32 * PLE_MAX_GATES), ("gate_input", c_int32 * PLE_MAX_GATES),
                ("gate_num_experts", c_int32 * PLE_MAX_GATES),
                ("gate_experts", (ctypes.c_uint8 * PLE_MAX_GATE_EXPERTS) * PLE_MAX_GATES),
                ("experts", c_void_p * PLE_MAX_EXPERTS), ("inputs", c_void_p * PLE_MAX_GATES),
                ("weight", c_void_p * PLE_MAX_GATES), ("bias", c_void_p * PLE_MAX_GATES),
                ("d_inputs", c_void_p * PLE_MAX_GATES)]


PEPNET_MAX_SEGS, PEPNET_IDENTITY, PEPNET_RELU = 8, 0, 1


class TzkPepnetSeg(ctypes.Structure):
    """struct tzk_pepnet_seg (include/tzk.h): one [B, N] segment of the PEPNet gate product."""

    _fields_ = [("x", c_void_p), ("bx", c_void_p), ("z", c_void_p), ("bz", c_void_p), ("y", c_void_p),
                ("dy", c_void_p), ("dx", c_void_p), ("dz", c_void_p), ("ldx", c_int64), ("ldz", c_int64),
                ("ldy", c_int64), ("N", c_int32), ("act", c_int32), ("gamma", c_float), ("pad_", c_int32)]


class TzkPepnetGateArgs(ctypes.Structure):
    """struct tzk_pepnet_gate_args (include/tzk.h): up to 8 segments sharing the batch size."""

    _fields_ = [("B", c_int64), ("n_segs", c_int32), ("pad_", c_int32), ("seg", TzkPepnetSeg * PEPNET_MAX_SEGS)]


ROCKET_MAX_PAIRS, ROCKET_MAX_CLASSES, ROCKET_COSINE, ROCKET_EUCLID = 8, 8, 0, 1


class TzkRocketHead(ctypes.Structure):
    """struct tzk_rocket_head (include/tzk.h): one output head of RocketLaunching (hidden, Linear, logits, probs)."""

    _fields_ = [("h", c_void_p), ("w", c_void_p), ("b", c_void_p), ("logits", c_void_p), ("probs", c_void_p),
                ("dh", c_void_p), ("H", c_int32), ("pad_", c_int32)]


class TzkRocketPair(ctypes.Structure):
    """struct tzk_rocket_pair (include/tzk.h): one light / booster hidden-layer pair of the similarity losses."""

    _fields_ = [("light", c_void_p), ("booster", c_void_p), ("dlight", c_void_p), ("d", c_int32), ("pad_", c_int32)]


class TzkRocketArgs(ctypes.Structure):
    """struct tzk_rocket_args (include/tzk.h): the light head, optionally the booster head and up to 8 pairs."""

    _fields_ = [("B", c_int64), ("C", c_int32), ("has_booster", c_int32), ("n_pairs", c_int32), ("sim", c_int32),
                ("eps", c_float), ("pad_", c_int32), ("labels", c_void_p), ("pair_stats", c_void_p),
                ("head", TzkRocketHead * 2), ("pair", TzkRocketPair * ROCKET_MAX_PAIRS)]


TDM_MAX_LAYERS, TDM_MAX_WINDOWS, TDM_RELU, TDM_PRELU = 3, 32, 0, 1


class TzkTdmArgs(ctypes.Structure):
    """struct tzk_tdm_args (include/tzk.h): TDM's multi-window DIN attention over jagged rows."""

    _fields_ = [("B", c_int64), ("N", c_int64), ("C", c_int32), ("Dq", c_int32), ("L", c_int32), ("n_layers", c_int32),
                ("act", c_int32), ("pad_", c_int32), ("windows", c_int32 * TDM_MAX_WINDOWS),
                ("hidden", c_int32 * TDM_MAX_LAYERS), ("pad2_", c_int32), ("seq", c_void_p), ("offsets", c_void_p),
                ("query", c_void_p), ("w", c_void_p * TDM_MAX_LAYERS), ("b", c_void_p * TDM_MAX_LAYERS),
                ("slope", c_void_p * TDM_MAX_LAYERS), ("lin_w", c_void_p), ("lin_b", c_void_p), ("act_w", c_void_p),
                ("out", c_void_p), ("z", c_void_p), ("d_out", c_void_p), ("d_seq", c_void_p), ("d_query", c_void_p)]


DCN_V2_MAX_LAYERS = 8


class TzkDcnV2Args(ctypes.Structure):
    """struct tzk_dcn_v2_args (include/tzk.h): DCN-v2's low-rank cross network."""

    _fields_ = [("B", c_int64), ("D", c_int32), ("L", c_int32), ("r", c_int32), ("pad_", c_int32), ("x0", c_void_p),
                ("wu", c_void_p), ("wv", c_void_p), ("bias", c_void_p), ("work", c_void_p), ("y", c_void_p),
                ("v", c_void_p), ("dy", c_void_p), ("dx0", c_void_p), ("dv", c_void_p)]


class TzkSeqAttnArgs(ctypes.Structure):
    """struct tzk_seq_attn_args (include/tzk.h): SelfAttentionEncoder's attention core over jagged rows."""

    _fields_ = [("B", c_int64), ("N", c_int64), ("H", c_int32), ("hd", c_int32), ("max_len", c_int32),
                ("pad_", c_int32), ("ldq", c_int64), ("ldk", c_int64), ("ldv", c_int64), ("offsets", c_void_p),
                ("q", c_void_p), ("k", c_void_p), ("v", c_void_p), ("pooled", c_void_p), ("lse", c_void_p),
                ("d_pooled", c_void_p), ("dq", c_void_p), ("dk", c_void_p), ("dv", c_void_p), ("dsum", c_void_p)]


class TzkJaggedPoolArgs(ctypes.Structure):
    """struct tzk_jagged_pool_args (include/tzk.h): PoolingEncoder over jagged rows."""

    _fields_ = [("B", c_int64), ("N", c_int64), ("D", c_int32), ("max_len", c_int32), ("mean", c_int32),
                ("pad_", c_int32), ("offsets", c_void_p), ("seq", c_void_p), ("out", c_void_p), ("d_out", c_void_p),
                ("d_seq", c_void_p)]


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
    "tzk_interact_wide_bwd_scaled": (
        c_int32, [P, c_int64, P, P, c_int64, P, c_int64, P, c_int64, c_int64, P, c_int64, P, c_int64, P, P, P]),
    "tzk_interact_wide_fwd": (
        c_int32, [P, c_int64, P, c_int64, P, c_int64, P, c_int64, P, c_int64, P, c_int64, P, P, P]),
    "tzk_interact_wide_wgrad": (
        c_int32, [P, c_int64, P, c_int64, P, c_int64, P, c_int64, c_int64, c_int32, P, P, c_int64, P]),
    "tzk_interact_wide_wgrad_scaled": (
        c_int32, [P, c_int64, P, P, c_int64, P, c_int64, P, c_int64, c_int64, c_int32, P, P, c_int64, P]),
    "tzk_tower_tail_bce_workspace_bytes": (c_size_t, [c_int64, c_int32, c_int32]),
    "tzk_tower_tail_bce": (
        c_int32, [P, c_int64, P, P, P, P, P, c_int64, c_int32, c_int32, P, P, c_int64, P, P, P, c_size_t, P]),
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
    "tzk_binned_auc_update": (c_int32, [P, c_int32, P, c_int32, c_int64, P, c_int32, P, P, P]),
    # FP16 tables on the peer step: the fp32 entry points' arguments, arenas and mirror of halfs
    "tzk_peer_pooled_gather_fwd_f16": (
        c_int32, [P, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P, P, P]),
    "tzk_peer_pooled_gather_fwd_sel_f16": (
        c_int32, [P, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P, P, P, c_int32, P]),
    "tzk_peer_pooled_gather_fwd_weighted_f16": (
        c_int32, [P, P, P, P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, P, c_int64, P, P, P, P, c_int32, P]),
    "tzk_peer_seq_gather_fwd_f16": (
        c_int32, [P, P, P, P, P, P, P, c_int32, c_int32, c_int32, c_int32, c_int64, P, P, P, P]),
    "tzk_peer_mirror_refresh_f16": (c_int32, [P, c_int32, P, P, P, P, c_int32, P, P]),
    # WuKong layer: the FM / linear-compress mix and the output norm, forward and backward
    "tzk_wukong_mix_fwd": (
        c_int32, [P, P, P, P, P, P, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, P, P, P, P]),
    "tzk_wukong_mix_bwd": (
        c_int32,
        [P, P, P, P, P, P, P, P, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32, P, P, P, P]),
    "tzk_wukong_out_fwd": (c_int32, [P, P, P, P, c_int64, c_int32, c_int32, c_int32, c_int32, P, P, P]),
    "tzk_wukong_out_bwd": (
        c_int32, [P, P, P, P, P, c_int64, c_int32, c_int32, c_int32, c_int32, P, P, P, P, P]),
    # MaskNet: the instance-guided mask and the FFN's bias + LayerNorm + ReLU, forward and backward
    "tzk_masknet_mask_fwd": (c_int32, [P, c_int32, P, P, P, P, c_int64, c_int32, c_int32, c_int32, P, P, P]),
    "tzk_masknet_mask_bwd": (
        c_int32, [P, c_int32, P, P, P, P, P, P, c_int64, c_int32, c_int32, c_int32, P, P, P, P, P]),
    "tzk_masknet_ffn_fwd": (c_int32, [P, P, P, P, c_int64, c_int32, c_int32, c_int32, P, P, P]),
    "tzk_masknet_ffn_bwd": (c_int32, [P, P, P, P, P, P, c_int64, c_int32, c_int32, c_int32, P, P, P, P]),
    # PLE: every gate of one extraction layer, forward and backward (the layer described by TzkPleGateArgs)
    "tzk_ple_gate_smem_bytes": (c_int64, [P, c_int32]),
    "tzk_ple_gate_fwd": (c_int32, [P, c_int32, P, P, P]),
    "tzk_ple_gate_bwd": (c_int32, [P, P, P, c_int32, P, P, P, P]),
    # PEPNet: the gate-neural-unit product of up to 8 segments (the segments described by TzkPepnetGateArgs)
    "tzk_pepnet_gate_fwd": (c_int32, [P, c_int32, P]),
    "tzk_pepnet_gate_bwd": (c_int32, [P, c_int32, P, P, P]),
    # JRC loss: session sort, per-session sums, loss and d loss / d logits in one call
    "tzk_jrc_loss_workspace_bytes": (c_size_t, [c_int64]),
    "tzk_jrc_loss": (c_int32, [P, c_int64, P, P, P, c_int64, c_float, c_int32, P, P, P, c_size_t, P]),
    # RocketLaunching: both output heads, their softmax and every distillation loss (TzkRocketArgs), each direction
    "tzk_rocket_head_fwd": (c_int32, [P, c_int32, P, P, P]),
    "tzk_rocket_head_bwd": (c_int32, [P, P, P, c_int32, P, P, P]),
    # TDM: the multi-window DIN attention over jagged rows (TzkTdmArgs), each direction
    "tzk_tdm_smem_bytes": (c_int64, [P, c_int32]),
    "tzk_tdm_fwd": (c_int32, [P, c_int32, P]),
    "tzk_tdm_bwd": (c_int32, [P, c_int32, P, P, P]),
    # DCN-v2: the low-rank cross network (TzkDcnV2Args), forward, input gradient and weight gradient
    "tzk_dcn_v2_smem_bytes": (c_int64, [P, c_int32]),
    "tzk_dcn_v2_fwd": (c_int32, [P, c_int32, P]),
    "tzk_dcn_v2_bwd_data": (c_int32, [P, c_int32, P]),
    "tzk_dcn_v2_bwd_weight": (c_int32, [P, c_int32, P, P, P]),
    # sequence encoders of DEEP groups: the self-attention core (TzkSeqAttnArgs) and the pooling encoder
    # (TzkJaggedPoolArgs) over jagged rows, each direction
    "tzk_seq_attn_smem_bytes": (c_int64, [P]),
    "tzk_self_attn_pool_fwd": (c_int32, [P, c_int32, P]),
    "tzk_self_attn_pool_bwd": (c_int32, [P, c_int32, P]),
    "tzk_jagged_pool_fwd": (c_int32, [P, c_int32, P]),
    "tzk_jagged_pool_bwd": (c_int32, [P, c_int32, P]),
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
