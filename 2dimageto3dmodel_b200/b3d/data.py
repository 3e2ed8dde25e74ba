"""Binding of b3d_gather_fields: one launch that assembles a batch from packed per-record stores (gather by index,
fp16 -> fp32, UV mirroring).  The stores may sit in device memory or in pinned host memory (read over PCIe)."""
import ctypes

import torch

from . import B3DError, check, lib, ptr, stream_ptr

F32, F16, I64 = 0, 1, 2
MAX_FIELDS = 8
_TYPES = {torch.float32: F32, torch.float16: F16, torch.int64: I64}


class GatherField(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("src_type", ctypes.c_int), ("n", ctypes.c_int), ("C_src", ctypes.c_int),
                ("C", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("mirror", ctypes.c_int),
                ("scale", ctypes.c_float), ("bias", ctypes.c_float), ("dst", ctypes.c_void_p)]


def _as4(shape):
    """[n, C, H, W] or [n, K] (rows of K, e.g. class labels) -> (n, C, H, W)."""
    if len(shape) == 4:
        return tuple(shape)
    if len(shape) == 2:
        return shape[0], shape[1], 1, 1
    raise B3DError(f"gather: expected a [n,C,H,W] or [n,K] store, got shape {tuple(shape)}")


def gather_fields(fields, idx, flip=None):
    """fields: list of (src, dst, mirror, scale, bias).  src [n,C_src,H,W] fp16 / fp32 (or [n,K] int64), contiguous, on
    the device or in pinned host memory; dst [B,C,H,W] fp32 (int64 [B,K]) on the device, C <= C_src.
    idx: int32 [B] CUDA tensor of record indices; flip: uint8 [B] CUDA tensor or None.
    dst[b,c] = scale * src[idx[b], c] + bias, mirrored in u where mirror and flip[b] are set."""
    if not 1 <= len(fields) <= MAX_FIELDS:
        raise B3DError(f"gather: 1 to {MAX_FIELDS} fields, got {len(fields)}")
    if not (isinstance(idx, torch.Tensor) and idx.is_cuda and idx.dtype == torch.int32 and idx.dim() == 1
            and idx.is_contiguous()):
        raise B3DError("gather: idx must be a contiguous int32 CUDA tensor [B]")
    B = idx.shape[0]
    if flip is not None and not (isinstance(flip, torch.Tensor) and flip.is_cuda and flip.dtype == torch.uint8
                                 and tuple(flip.shape) == (B,) and flip.is_contiguous()):
        raise B3DError("gather: flip must be a contiguous uint8 CUDA tensor [B] or None")
    arr = (GatherField * len(fields))()
    for i, (src, dst, mirror, scale, bias) in enumerate(fields):
        if src.dtype not in _TYPES:
            raise B3DError(f"gather: field {i}: store dtype {src.dtype} (expected float16, float32 or int64)")
        want = torch.int64 if src.dtype == torch.int64 else torch.float32
        if dst.dtype != want or not dst.is_cuda:
            raise B3DError(f"gather: field {i}: output must be a {want} CUDA tensor, got {dst.dtype} on {dst.device}")
        if not (src.is_contiguous() and dst.is_contiguous()):
            raise B3DError(f"gather: field {i}: store and output must be contiguous")
        n, C_src, H, W = _as4(src.shape)
        Bd, C, Hd, Wd = _as4(dst.shape)
        if (Bd, Hd, Wd) != (B, H, W) or C > C_src:
            raise B3DError(f"gather: field {i}: output {tuple(dst.shape)} does not fit store {tuple(src.shape)} and B={B}")
        arr[i] = GatherField(src.data_ptr(), _TYPES[src.dtype], n, C_src, C, H, W, int(bool(mirror)), float(scale),
                             float(bias), dst.data_ptr())
    check(lib.b3d_gather_fields(ctypes.cast(arr, ctypes.c_void_p), len(fields), ptr(idx), ptr(flip), B, stream_ptr(idx)))
