"""Host-side mirror of libavcodec's HEVC motion compensation: the put_hevc_{q,e}pel tables of HEVCDSPContext as ff_hevc_dsp_init
installs them (libavcodec/hevc/dsp.c:140-196), and the batched device entry b200_hevc_mc_batch_device."""
import ctypes as C

import numpy as np

from ._lib import lib, check, vp, HEVCDSPContext, HevcMcOp

UNI, UNI_W, BI, BI_W = range(4)                 # B200HevcMcOp.kind
OP_DTYPE = np.dtype([("dst_off", "<i8"), ("ref_off", "<i8", 2), ("x", "<i4", 2), ("y", "<i4", 2), ("mx", "u1", 2), ("my", "u1", 2),
                     ("w", "u1"), ("h", "u1"), ("kind", "u1"), ("denom", "u1"), ("wx0", "<i4"), ("wx1", "<i4"), ("ox", "<i4"),
                     ("reserved", "u1", 4)])
assert OP_DTYPE.itemsize == C.sizeof(HevcMcOp) == 64


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_hevc_dsp_init(bit_depth=8):
    """HEVCDSPContext with the six inter-prediction tables filled (HOST pointers), every other member NULL"""
    c = HEVCDSPContext()
    check(lib().b200_hevc_dsp_init(C.byref(c), bit_depth), "ff_hevc_dsp_init")
    return c


def hevc_mc_batch_device(device, bit_depth, epel, nops, ops, dst, dst_stride, ref, ref_stride, pic_w, pic_h):
    """one plane's prediction units; ops = OP_DTYPE records (a uint8 tensor of nops * 64 bytes), dst / ref sample tensors, strides in
    bytes (device)"""
    return check(lib().b200_hevc_mc_batch_device(device.handle, bit_depth, epel, nops, vp(_dptr(ops)), vp(_dptr(dst)), dst_stride,
                                                 vp(_dptr(ref)), ref_stride, pic_w, pic_h), "hevc_mc_batch_device")
