"""Thin tensor-level wrappers over the T2I-Adapter's C-ABI entry points (csrc/adapter.cu), as mos_b200/ops.py does for
the rest of the library.  Every call here is audited by tests/adapter_audit.py (tests/test_adapter_audit_coverage.py keeps
the two in step).  Tensors are CUDA tensors owned by the caller; outputs are passed in."""
import ctypes

import torch

from . import _lib
from ._lib import act_dtype, check, current_stream, ptr


def _dt(*tensors):
    return ctypes.c_int32(act_dtype(*tensors))


def pixel_unshuffle(x, y, *, ldy=None):
    """fp32 NCHW image [B, Cin, H, W] -> 16-bit rows [B*(H/8)*(W/8), ldy], column c*64 + i*8 + j = x[b, c, 8h+i, 8w+j]"""
    assert x.dtype == torch.float32
    B, Cin, H, W = x.shape
    check(_lib.lib().mos_pixel_unshuffle(ptr(x), ctypes.c_int32(B), ctypes.c_int32(Cin), ctypes.c_int32(H),
                                         ctypes.c_int32(W), ptr(y), ctypes.c_int64(y.stride(0) if ldy is None else ldy),
                                         _dt(y), current_stream()), 'mos_pixel_unshuffle')
    return y


def relu_rows(x, *, M, C, ld=None):
    """x[m, :C] <- (x < 0 ? 0 : x) in place"""
    check(_lib.lib().mos_relu_rows(ptr(x), ctypes.c_int64(x.stride(0) if ld is None else ld), ctypes.c_int64(M),
                                   ctypes.c_int32(C), _dt(x), current_stream()), 'mos_relu_rows')
    return x


def avgpool2x(x, y, *, B, H, W, C, ldx=None, ldy=None):
    """NHWC [B, H, W, C] (pixel pitch ldx) -> [B, H/2, W/2, C] (pitch ldy): AvgPool2d(2, 2)"""
    check(_lib.lib().mos_avgpool2x(ptr(x), ctypes.c_int64(x.stride(-2) if ldx is None else ldx), ctypes.c_int32(B),
                                   ctypes.c_int32(H), ctypes.c_int32(W), ctypes.c_int32(C), ptr(y),
                                   ctypes.c_int64(y.stride(-2) if ldy is None else ldy), _dt(x, y), current_stream()),
          'mos_avgpool2x')
    return y
