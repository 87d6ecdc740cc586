"""fp32 Linear for the dense towers: hand-written kernels for the small layers (csrc/tzk_tower.cu) and the wide
783 -> 64 layer (csrc/tzk_gemm3x.cu), cuBLASLt (csrc/tzk_gemm.cpp) for the rest.

The towers are caller code (plain PyTorch in the reference, tzrec/modules/mlp.py); this only swaps the GEMM
algorithm: same fp32 inputs/outputs, fp32-equivalent accuracy.  cuBLASLt (>= 12.9) is asked for the BF16x9-emulated
fp32 compute type and for plain fp32 when it offers no algorithm for that; which kernels it runs is its choice per GPU.
Falls back to torch.nn.functional.linear whenever the library or the device is unavailable (set TZK_DENSE_GEMM=torch to force
the fallback).

Under torch.autocast (train_config.mixed_precision) the fp32 GEMM kernels step aside: `linear` is autocast's own F.linear
(lower-precision list), the fused interaction + wide layer and the fused tower tail give way to the layer-by-layer torch
chain, and the BCE kernel stays (autocast runs BCE-with-logits in fp32).  DLRM-Criteo's interaction under bf16 autocast
has a kernel of its own, InteractBf16Fn.
"""

import ctypes
import os
from typing import Optional

import torch
from torch import nn

from .functional import autocast_dtype

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "csrc", "libtzk_gemm.so")
_CUBLASLT_CANDIDATES = ["/usr/local/cuda/lib64/libcublasLt.so.12", "/usr/local/cuda-12.9/lib64/libcublasLt.so.12"]
_state = {"lib": None, "version": 0, "tried": False, "ws": {}, "emulated_calls": 0, "plain_calls": 0}


def _load():
    if _state["tried"]:
        return _state["lib"]
    _state["tried"] = True
    if os.environ.get("TZK_DENSE_GEMM", "") == "torch" or not os.path.exists(_LIB_PATH) or not torch.cuda.is_available():
        return None
    try:
        lib = ctypes.CDLL(_LIB_PATH)
        lib.tzg_init.restype = ctypes.c_long
        lib.tzg_init.argtypes = [ctypes.c_char_p]
        lib.tzg_last_error.restype = ctypes.c_char_p
        P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        lib.tzg_matmul.argtypes = [I, I, I, I, I, P, I, P, I, P, I, F, F, I, P, ctypes.c_size_t, P,
                                   ctypes.POINTER(ctypes.c_int)]
        for path in _CUBLASLT_CANDIDATES:
            if os.path.exists(path):
                v = lib.tzg_init(path.encode())
                if v >= 120900:      # BF16x9 emulation exists from cuBLAS 12.9 on
                    _state["lib"], _state["version"] = lib, v
                    break
    except OSError:
        _state["lib"] = None
    return _state["lib"]


def available() -> bool:
    return _load() is not None


def stats():
    return {"cublaslt": _state["version"], "emulated_calls": _state["emulated_calls"],
            "plain_calls": _state["plain_calls"]}


def _workspace(device) -> torch.Tensor:
    ws = _state["ws"].get(device)
    if ws is None:
        ws = torch.empty(64 << 20, dtype=torch.uint8, device=device)
        _state["ws"][device] = ws
    return ws


def _mm(a: torch.Tensor, ta: bool, b: torch.Tensor, tb: bool, M: int, N: int, K: int) -> torch.Tensor:
    """Row-major C[M,N] = op(a) @ op(b) through cuBLASLt BF16x9."""
    lib = _state["lib"]
    out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    ws = _workspace(a.device)
    used = ctypes.c_int(0)
    rc = lib.tzg_matmul(int(ta), int(tb), M, N, K, a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                        out.data_ptr(), N, 1.0, 0.0, 1, ws.data_ptr(), ws.numel(),
                        torch.cuda.current_stream().cuda_stream, ctypes.byref(used))
    if rc != 0:
        raise RuntimeError(lib.tzg_last_error().decode())
    _state["emulated_calls" if used.value else "plain_calls"] += 1
    return out


class _LinearFn(torch.autograd.Function):
    """y = act(x @ W^T + b), act = ReLU or identity (tzrec/modules/mlp.py Perceptron).  GEMMs: cuBLASLt BF16x9;
    bias+ReLU and ReLU-backward+bias-gradient are one tzk kernel each instead of four ATen passes.
    `x` may carry zero columns beyond W's in_features (width rounded up to a multiple of 4 by the producer):
    16-B aligned rows are what lets cuBLASLt pick the tensor-core kernels instead of the align1 SIMT ones —
    e.g. DLRM's 783-wide final-MLP input travels as [B, 784].  fp32 only: under autocast `linear` runs autocast's
    F.linear instead."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu, in_map):
        from .kernels import default_kernels

        K, Kx = weight.shape[1], x.shape[1]
        w = weight
        if Kx != K:      # zero-padded input: pad the weight the same way (N x Kx, a few hundred KB)
            w = torch.zeros((weight.shape[0], Kx), dtype=weight.dtype, device=weight.device)
            for (src, dst, n) in (in_map or ((0, 0, K),)):
                w[:, dst:dst + n].copy_(weight[:, src:src + n])
        ctx.in_map = in_map
        y = _mm(x, False, w, True, x.shape[0], w.shape[0], Kx)
        if bias is not None or relu:
            default_kernels().bias_act(y, bias, relu)
        ctx.save_for_backward(x, w, y if relu else None)
        ctx.has_bias, ctx.relu, ctx.K = bias is not None, relu, K
        return y

    @staticmethod
    def backward(ctx, dy):
        from .kernels import default_kernels

        x, w, y = ctx.saved_tensors
        dy = dy if (dy.stride(1) == 1 and dy.stride(0) >= dy.shape[1]) else dy.contiguous()
        N = w.shape[0]
        dx = dw = db = None
        fused = (256 % N == 0) and (ctx.has_bias or ctx.relu)
        if fused:       # dz = dy * (y > 0) and db = sum_rows(dz) in one pass
            dz, colsum = default_kernels().act_bwd_colsum(dy, y, ctx.relu, want_dz=ctx.relu)
            if not ctx.relu:
                dz = dy.contiguous()
            db = colsum if ctx.has_bias else None
        else:
            dz = dy * (y > 0) if ctx.relu else dy.contiguous()
            db = dz.sum(0) if ctx.has_bias else None
        if ctx.needs_input_grad[0]:
            dx = _mm(dz, False, w, False, dz.shape[0], w.shape[1], N)
        if ctx.needs_input_grad[1]:
            dw = _mm(dz, True, x, False, N, w.shape[1], dz.shape[0])
            if w.shape[1] != ctx.K:
                segs = ctx.in_map or ((0, 0, ctx.K),)
                dw = torch.cat([dw[:, dst:dst + n] for (_, dst, n) in segs], dim=1) if len(segs) > 1 \
                    else dw[:, :ctx.K].contiguous()
        if not ctx.needs_input_grad[2]:
            db = None
        return dx, dw, db, None, None


class _SmallLinearFn(torch.autograd.Function):
    """y = act(x @ W^T + b) for K, N <= 64: one tzk launch forward, one (+ partial reduction) backward
    (csrc/tzk_tower.cu) instead of the 4-10 library launches such a layer costs as GEMM + element-wise passes.
    fp32 only: under autocast `linear` runs autocast's F.linear instead."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        from .kernels import default_kernels

        w = weight.contiguous()
        y = default_kernels().small_linear_fwd(x, w, bias, relu)
        ctx.save_for_backward(x, w, y if relu else None)
        ctx.relu, ctx.has_bias = relu, bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        from .kernels import default_kernels

        x, w, y = ctx.saved_tensors
        dy = dy if (dy.stride(1) == 1 and dy.stride(0) >= dy.shape[1]) else dy.contiguous()
        dx, dw, db = default_kernels().small_linear_bwd(
            x, w, y, dy, ctx.relu, want_dx=ctx.needs_input_grad[0],
            want_db=ctx.has_bias and ctx.needs_input_grad[2])
        return dx, (dw if ctx.needs_input_grad[1] else None), db, None


# --------------------------------------------------------------------------------------------------------------------
# The one wide layer (N = 64 outputs, input width a multiple of 112: DLRM's 783-wide final-MLP input travels as
# [B, 784]) on hand-written TMA + mma.sync 3xTF32 kernels (csrc/tzk_gemm3x.cu -> libtzk_gemm3x.so): forward with bias + ReLU
# in the epilogue, dgrad on W^T, wgrad with a fixed-order slab reduction.  TZK_GEMM3X=1 selects it.
# --------------------------------------------------------------------------------------------------------------------
_G3 = {"lib": None, "tried": False}


def _gemm3x_lib():
    if not _G3["tried"]:
        _G3["tried"] = True
        path = os.path.join(_HERE, "csrc", "libtzk_gemm3x.so")
        if os.path.exists(path) and torch.cuda.is_available():
            _G3["lib"] = _declare_gemm3x(ctypes.CDLL(path))
    return _G3["lib"]


SLABS = 37          # 7 column tiles x 37 row slabs = 259 CTAs: two per SM of an H100 (132 SMs)


def _declare_gemm3x(L):
    P, I64, I32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
    L.tzk_gemm3x.argtypes = [P, I64, P, I64, P, I64, I32, I32, I32, P, I64, P, P, P]
    L.tzk_wgrad3x.argtypes = [P, I64, P, I64, I64, I32, I32, P, P, I64, P]
    L.tzk_wgrad3x_partial_floats.restype = I64
    L.tzk_wgrad3x_partial_floats.argtypes = [I32, I32]
    return L


def gemm3x_supported(M: int, N: int, Kx: int) -> bool:
    return N == 64 and Kx % 112 == 0 and Kx % 4 == 0 and M >= 1


def _g3_stream(t: torch.Tensor):
    return torch.cuda.current_stream().cuda_stream if t.is_cuda else None


def _g3_check(rc, what):
    if rc:
        raise RuntimeError(f"{what} failed with code {rc}")


def gemm3x(lib, x, w, bias, relu):
    """act(x [M, K] @ w [N, K]^T + bias) -> [M, N]; x rows may be strided (ld = x.stride(0))."""
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty((M, N), dtype=torch.float32, device=x.device)
    w_hi, w_lo = torch.empty_like(w), torch.empty_like(w)
    _g3_check(lib.tzk_gemm3x(x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), None if bias is None else bias.data_ptr(),
                          M, N, K, int(relu), y.data_ptr(), N, w_hi.data_ptr(), w_lo.data_ptr(), _g3_stream(x)), "tzk_gemm3x")
    return y


def wgrad3x(lib, x, dz, slabs=SLABS):
    """dz [M, 64]^T @ x [M, K] -> [64, K]."""
    M, K = x.shape
    dw = torch.empty((64, K), dtype=torch.float32, device=x.device)
    part = torch.empty(lib.tzk_wgrad3x_partial_floats(K, slabs), dtype=torch.float32, device=x.device)
    _g3_check(lib.tzk_wgrad3x(x.data_ptr(), x.stride(0), dz.data_ptr(), dz.stride(0), M, K, slabs, part.data_ptr(),
                           dw.data_ptr(), K, _g3_stream(x)), "tzk_wgrad3x")
    return dw


class Gemm3xLinearFn(torch.autograd.Function):
    """Same contract as dense_gemm._LinearFn.apply(x, weight, bias, relu, in_map) with `lib` in front.  fp32 only: under
    autocast `linear` runs autocast's F.linear instead."""

    @staticmethod
    def forward(ctx, lib, x, weight, bias, relu, in_map):
        K, Kx = weight.shape[1], x.shape[1]
        w = weight.contiguous()
        if Kx != K:      # zero-padded / column-mapped input: lay the weight out the same way
            w = torch.zeros((weight.shape[0], Kx), dtype=weight.dtype, device=weight.device)
            for (src, dst, n) in (in_map or ((0, 0, K),)):
                w[:, dst:dst + n].copy_(weight[:, src:src + n])
        if not gemm3x_supported(x.shape[0], w.shape[0], Kx):
            raise ValueError(f"gemm3x covers N = 64 and input widths that are multiples of 112, got {tuple(w.shape)}")
        y = gemm3x(lib, x, w, bias, relu)
        ctx.lib, ctx.in_map, ctx.K = lib, in_map, K
        ctx.has_bias, ctx.relu = bias is not None, relu
        ctx.save_for_backward(x, w, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        lib = ctx.lib
        if dy.is_cuda and (ctx.has_bias or ctx.relu):
            from .kernels import default_kernels

            dz, colsum = default_kernels().act_bwd_colsum(dy.contiguous(), y, ctx.relu, want_dz=ctx.relu)
            dz = dz if ctx.relu else dy.contiguous()
            db = colsum if ctx.has_bias else None
        else:
            dz = (dy * (y > 0) if ctx.relu else dy).contiguous()
            db = dz.sum(0) if ctx.has_bias else None
        dx = dw = None
        if ctx.needs_input_grad[1]:
            dx = gemm3x(lib, dz, w.t().contiguous(), None, False)            # [M, 64] x [Kx, 64]^T
        if ctx.needs_input_grad[2]:
            dw = wgrad3x(lib, x, dz)
            if w.shape[1] != ctx.K:
                segs = ctx.in_map or ((0, 0, ctx.K),)
                dw = torch.cat([dw[:, dst:dst + n] for (_, dst, n) in segs], dim=1) if len(segs) > 1 \
                    else dw[:, :ctx.K].contiguous()
        if not ctx.needs_input_grad[3]:
            db = None
        return None, dx, dw, db, None, None


class InteractWideFn(torch.autograd.Function):
    """relu(X @ W^T + b) with X = functional.dlrm_interaction(dense, sparse, 26, 16, aligned=True), the first layer of
    DLRM-Criteo's final MLP.  The forward is the interaction kernel followed by gemm3x; the backward computes the
    interaction's input gradients in one kernel from dZ and W (tzk_interact_wide_bwd) instead of writing X's gradient
    [M, 784] to memory and reading it back, and the weight gradient with wgrad3x from the saved X.  fp32 only: under
    autocast interact_wide_usable() is False and the layer runs as autocast's F.linear."""

    @staticmethod
    def forward(ctx, lib, dense, sparse, weight, bias, in_map):
        from .functional import _rows_contig, backend

        dense, sparse = _rows_contig(dense), _rows_contig(sparse)
        x = backend().dot_interact_fwd(dense, sparse, 26, 16, True, True, 4, 1)
        w = torch.zeros((weight.shape[0], x.shape[1]), dtype=weight.dtype, device=weight.device)
        for (src, dst, n) in in_map:
            w[:, dst:dst + n].copy_(weight[:, src:src + n])
        y = gemm3x(lib, x, w, bias, True)
        ctx.lib, ctx.in_map, ctx.has_bias = lib, in_map, bias is not None
        ctx.save_for_backward(dense, sparse, x, w, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        from .kernels import default_kernels

        dense, sparse, x, w, y = ctx.saved_tensors
        lib = ctx.lib
        dz, colsum = default_kernels().act_bwd_colsum(dy.contiguous(), y, True, want_dz=True)
        d_dense = d_sparse = dw = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            d_dense, d_sparse = default_kernels().interact_wide_bwd(dz, w, dense, sparse)
        if ctx.needs_input_grad[3]:
            full = wgrad3x(lib, x, dz)
            dw = torch.cat([full[:, dst:dst + n] for (_, dst, n) in ctx.in_map], dim=1)
        db = colsum if (ctx.has_bias and ctx.needs_input_grad[4]) else None
        return (None, d_dense if ctx.needs_input_grad[1] else None, d_sparse if ctx.needs_input_grad[2] else None, dw, db,
                None)


class InteractBf16Fn(torch.autograd.Function):
    """X [B, 784] bf16 = [351 pairs | 0 | dense | bf16(sparse)], DLRM-Criteo's interaction under bf16 autocast
    (csrc/tzk_interact_bf16.cuh), from the bottom MLP's bf16 output [B, 16] and the pooled embeddings [B, 416] fp32.  The
    rounding points are those of dlrm.py:113-131 under autocast: bf16 pairs from fp32 accumulation, bf16 copies, and in
    the backward d_dense in bf16 and d_sparse in fp32 (include/tzk.h).  The first final-MLP layer consumes X as autocast's
    F.linear with the weight spread by IN_MAP."""

    IN_MAP = ((0, 0, 351), (351, 352, 432))

    @staticmethod
    def forward(ctx, dense, sparse):
        from .kernels import default_kernels

        ctx.save_for_backward(dense, sparse)
        return default_kernels().dot_interact27_fwd_bf16(dense, sparse)

    @staticmethod
    def backward(ctx, dx):
        from .kernels import default_kernels

        dense, sparse = ctx.saved_tensors
        if not (dx.stride(1) == 1 and dx.stride(0) % 8 == 0 and dx.data_ptr() % 16 == 0):
            dx = dx.contiguous()
        d_dense, d_sparse = default_kernels().dot_interact27_bwd_bf16(dx, dense, sparse)
        return (d_dense if ctx.needs_input_grad[0] else None), (d_sparse if ctx.needs_input_grad[1] else None)


def interact_bf16_usable(dense: Optional[torch.Tensor], sparse: torch.Tensor, num_sparse: int, dim: int) -> bool:
    """Whether InteractBf16Fn covers this interaction: bf16 autocast on CUDA, DLRM-Criteo's shape (26 sparse features of
    16 plus a bf16 bottom-MLP output [B, 16]), rows aligned for the kernel's vector loads.  TZK_INTERACT_BF16=0 selects
    the torch formulation instead."""
    return (dense is not None and sparse.is_cuda and autocast_dtype(sparse) == torch.bfloat16 and num_sparse == 26
            and dim == 16 and dense.dtype == torch.bfloat16 and sparse.dtype == torch.float32 and dense.dim() == 2
            and sparse.dim() == 2 and tuple(dense.shape[1:]) == (16,) and tuple(sparse.shape[1:]) == (416,)
            and dense.shape[0] == sparse.shape[0] >= 1
            and dense.stride(1) == 1 and dense.stride(0) % 4 == 0 and dense.data_ptr() % 8 == 0
            and sparse.stride(1) == 1 and sparse.stride(0) % 4 == 0 and sparse.data_ptr() % 16 == 0
            and os.environ.get("TZK_INTERACT_BF16", "1") != "0")


def interact_wide_usable(dense: Optional[torch.Tensor], sparse: torch.Tensor, weight: torch.Tensor,
                         num_sparse: int, dim: int) -> bool:
    """Whether InteractWideFn covers this layer: DLRM-Criteo's shape (26 sparse features of 16 plus the bottom-MLP
    output, all copied into the row), fp32 CUDA tensors, a 783 -> 64 weight, and the kernels the layer-by-layer path
    would run (gemm3x for the layer, the tensor-core interaction), and autocast off."""
    return (dense is not None and autocast_dtype(sparse) is None and num_sparse == 26 and dim == 16 and dense.is_cuda and dense.dtype == torch.float32
            and sparse.dtype == torch.float32 and dense.dim() == 2 and tuple(dense.shape[1:]) == (16,)
            and sparse.dim() == 2 and tuple(sparse.shape[1:]) == (416,) and dense.shape[0] == sparse.shape[0] >= 256
            and all(t.stride(1) == 1 and t.stride(0) % 4 == 0 and t.data_ptr() % 16 == 0 for t in (dense, sparse))
            and weight.dtype == torch.float32 and tuple(weight.shape) == (64, 783)
            and os.environ.get("TZK_GEMM3X", "1") == "1" and os.environ.get("TZK_INTERACT_TC", "1") != "0"
            and os.environ.get("TZK_INTERACT_TC_FWD", "1") != "0" and os.environ.get("TZK_INTERACT_TC_BWD", "1") != "0"
            and not torch.backends.cuda.matmul.allow_tf32 and available() and _gemm3x_lib() is not None)


def _use_gemm3x(x: torch.Tensor, weight: torch.Tensor) -> bool:
    return (os.environ.get("TZK_GEMM3X", "1") == "1" and x.is_cuda and x.dim() == 2 and x.dtype == torch.float32
            and weight.dtype == torch.float32 and x.stride(1) == 1 and x.stride(0) % 4 == 0 and x.data_ptr() % 16 == 0
            and gemm3x_supported(x.shape[0], weight.shape[0], x.shape[1]) and _gemm3x_lib() is not None)


SMALL_MAX = 64      # tzk_small_linear_*: K, N <= 64


def _small(x: torch.Tensor, weight: torch.Tensor) -> bool:
    return (x.is_cuda and x.dim() == 2 and x.dtype == torch.float32 and weight.dtype == torch.float32
            and weight.shape[0] <= SMALL_MAX and weight.shape[1] <= SMALL_MAX and x.shape[1] == weight.shape[1]
            and x.shape[0] >= 1 and x.stride(1) == 1 and x.stride(0) >= x.shape[1]
            and os.environ.get("TZK_SMALL_LINEAR", "1") != "0")


class _BceFn(torch.autograd.Function):
    """mean BCE-with-logits; the forward kernel also writes dloss/dlogits, backward only scales it.  Kept under autocast:
    binary_cross_entropy_with_logits is on autocast's fp32 list, so bce_with_logits() hands it fp32 logits."""

    @staticmethod
    def forward(ctx, logits, labels):
        from .kernels import default_kernels

        loss, dz = default_kernels().bce_logits_fwd_bwd(logits.contiguous(), labels.contiguous())
        ctx.save_for_backward(dz)
        ctx.shape = logits.shape
        return loss

    @staticmethod
    def backward(ctx, g):
        (dz,) = ctx.saved_tensors
        return (dz * g).view(ctx.shape), None


class _TowerTailFn(torch.autograd.Function):
    """(loss, logits) = BCE(Linear(relu(Linear(y1)))) with every gradient computed in the forward kernel.  fp32 only:
    under autocast tower_tail_usable() is False and the two layers run as autocast's F.linear."""

    @staticmethod
    def forward(ctx, y1, w1, b1, w2, b2, labels):
        from .kernels import default_kernels

        loss, logits, dy1, dw1, db1, dw2, db2 = default_kernels().tower_tail_bce(y1, w1, b1, w2, b2, labels)
        ctx.save_for_backward(dy1, dw1, db1, dw2, db2)
        ctx.has = (b1 is not None, b2 is not None)
        ctx.mark_non_differentiable(logits)
        return loss, logits

    @staticmethod
    def backward(ctx, g_loss, _g_logits):
        dy1, dw1, db1, dw2, db2 = ctx.saved_tensors
        # (g_loss is 1 in a plain `loss.backward()`; any other scale multiplies through)
        return (dy1 * g_loss, dw1 * g_loss, (db1 * g_loss) if ctx.has[0] else None, dw2 * g_loss,
                (db2 * g_loss) if ctx.has[1] else None, None)


def tower_tail_usable(y1: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, labels: torch.Tensor) -> bool:
    """The fused tail covers fp32 CUDA towers ending K -> N (ReLU) -> 1 with K, N <= 64 and a float label per row, with
    autocast off."""
    return (autocast_dtype(y1) is None and y1.is_cuda and y1.dim() == 2 and y1.dtype == torch.float32 and w1.dtype == torch.float32
            and w1.shape[1] == y1.shape[1] <= 64 and w1.shape[0] <= 64 and tuple(w2.shape) == (1, w1.shape[0])
            and labels.dtype == torch.float32 and labels.numel() == y1.shape[0] >= 1 and y1.stride(1) == 1)


def tower_tail_bce(y1, w1, b1, w2, b2, labels):
    """-> (mean BCE loss, logits [M]) of Linear(N, 1)(relu(Linear(K, N)(y1))) against `labels`."""
    return _TowerTailFn.apply(y1, w1, b1, w2, b2, labels)


def bce_with_logits(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """F.binary_cross_entropy_with_logits(logits, labels) (mean); fused fwd+bwd kernel on CUDA fp32 inputs.  Under
    autocast the logits are cast to fp32 first, as autocast's fp32 list does for this op."""
    if autocast_dtype(logits) is not None:
        logits, labels = logits.float(), labels.float()
    if (logits.is_cuda and logits.dtype == torch.float32 and labels.dtype == torch.float32 and logits.numel() >= 1
            and os.environ.get("TZK_SMALL_LINEAR", "1") != "0"):
        return _BceFn.apply(logits, labels)
    return torch.nn.functional.binary_cross_entropy_with_logits(logits, labels)


def _spread_weight(weight: torch.Tensor, width: int, in_map) -> torch.Tensor:
    """[N, K] -> [N, width]: column src of `weight` at column dst for every (src, dst, n) of `in_map` (default: the K
    columns first), zeros elsewhere; differentiable, so the gradient reaches `weight`."""
    N, K = weight.shape
    cols, c = [], 0
    for (src, dst, n) in (in_map or ((0, 0, K),)):
        if dst > c:
            cols.append(weight.new_zeros((N, dst - c)))
        cols.append(weight[:, src:src + n])
        c = dst + n
    if width > c:
        cols.append(weight.new_zeros((N, width - c)))
    return torch.cat(cols, dim=1)


def padded_width(n: int) -> int:
    return (n + 3) // 4 * 4


def _usable(x: torch.Tensor, weight: torch.Tensor) -> bool:
    return (x.is_cuda and x.dim() == 2 and x.dtype == torch.float32 and weight.dtype == torch.float32
            and x.shape[0] >= 256 and x.stride(1) == 1 and x.stride(0) >= x.shape[1]
            and not torch.backends.cuda.matmul.allow_tf32 and available())


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], relu: bool = False,
           in_map=None) -> torch.Tensor:
    """act(F.linear(x, weight, bias)).  `x` may be wider than in_features: zero-padded at the end (width =
    padded_width(in_features)) or, with `in_map` = ((src_col, dst_col, n), ...), with zero columns in between —
    column src of the weight multiplies column dst of x.

    Under autocast this is autocast's own F.linear (lower-precision list: inputs and weight cast, fp32 accumulation);
    a wider `x` meets the weight spread to its columns through differentiable ops, so the zero columns contribute
    nothing and the weight gradient is the reference's."""
    K = weight.shape[1]
    if autocast_dtype(x) is not None:
        if x.dim() == 2 and (x.shape[1] != K or in_map is not None):
            if in_map is None and x.shape[1] != padded_width(K):
                raise RuntimeError(f"linear: input width {x.shape[1]} does not match in_features {K}")
            weight = _spread_weight(weight, x.shape[1], in_map)
        y = torch.nn.functional.linear(x, weight, bias)
        return torch.relu(y) if relu else y
    if in_map is None and _small(x, weight):
        return _SmallLinearFn.apply(x, weight, bias, relu)
    if x.dim() == 2 and (x.shape[1] != K or in_map is not None):
        if in_map is None and x.shape[1] != padded_width(K):
            raise RuntimeError(f"linear: input width {x.shape[1]} does not match in_features {K}")
        if not _usable(x, weight):       # fallback: drop the padding columns
            x = x[:, :K] if in_map is None else torch.cat([x[:, d:d + n] for (_, d, n) in in_map], dim=1)
            in_map = None
    if _usable(x, weight):
        if _use_gemm3x(x, weight):
            return Gemm3xLinearFn.apply(_gemm3x_lib(), x, weight, bias, relu, in_map)
        return _LinearFn.apply(x, weight, bias, relu, in_map)
    y = torch.nn.functional.linear(x, weight, bias)
    return torch.relu(y) if relu else y


class Linear(nn.Linear):
    """nn.Linear whose 2-D fp32 CUDA GEMMs go through `linear`."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return linear(x, self.weight, self.bias)
