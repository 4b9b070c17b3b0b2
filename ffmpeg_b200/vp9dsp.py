"""Host-side mirror of libavcodec's VP9 DSP: the mc / smc tables of VP9DSPContext as ff_vp9dsp_init installs them
(libavcodec/vp9dsp_template.c:2302-2361, :2540-2569) and the batched device entry b200_vp9_mc_batch_device; the itxfm_add members
(vp9dsp_template.c:1755-1778) and b200_vp9_itxfm_add_batch_device; the loop-filter members (vp9dsp_template.c:1947-1967) and the frame
entry b200_vp9_loopfilter_frame_device (ff_vp9_loopfilter_sb over every superblock, vp9lpf.c:179-203); the intra_pred members
(vp9dsp_template.c:1120-1152) and the frame entry b200_vp9_intra_recon_frame_device (intra_recon over every intra transform block,
vp9recon.c:219-287)."""
import ctypes as C

import numpy as np

from ._lib import lib, check, vp, VP9DSPContext, Vp9McRef, Vp9McOp, VP9_MC_FUNC, VP9_SCALED_MC_FUNC, Vp9TxOp, VP9_ITXFM_FUNC, Vp9Filter, VP9_LF_FUNC, Vp9IntraOp, VP9_INTRA_FUNC  # noqa: F401

SINGLE, COMPOUND = range(2)                                          # B200Vp9McOp.kind
FILTER_8TAP_SMOOTH, FILTER_8TAP_REGULAR, FILTER_8TAP_SHARP, FILTER_BILINEAR = range(4)   # B200Vp9McOp.filter, libavcodec/vp9.h:64-71
MAX_REFS = 8
OP_DTYPE = np.dtype([("dst_off", "<i8"), ("x", "<i4", 2), ("y", "<i4", 2), ("ref", "u1", 2), ("mx", "u1", 2), ("my", "u1", 2),
                     ("w", "u1"), ("h", "u1"), ("filter", "u1"), ("kind", "u1"), ("reserved", "u1", 6)])
assert OP_DTYPE.itemsize == C.sizeof(Vp9McOp) == 40
DCT_DCT, DCT_ADST, ADST_DCT, ADST_ADST = range(4)                     # B200Vp9TxOp.type, libavcodec/vp9.h TxfmType
TX_4X4, TX_8X8, TX_16X16, TX_32X32, TX_LOSSLESS = range(5)            # B200Vp9TxOp.tx
TX_DTYPE = np.dtype([("dst_off", "<i8"), ("coef_off", "<i8"), ("tx", "u1"), ("type", "u1"), ("eob", "<u2"), ("reserved", "u1", 4)])
assert TX_DTYPE.itemsize == C.sizeof(Vp9TxOp) == 24
LF_DTYPE = np.dtype([("level", "u1", 64), ("mask", "u1", (2, 2, 8, 4))])    # B200Vp9Filter: [luma / chroma][column / row edges][row][width]
assert LF_DTYPE.itemsize == C.sizeof(Vp9Filter) == 192
(VERT_PRED, HOR_PRED, DC_PRED, DIAG_DOWN_LEFT_PRED, DIAG_DOWN_RIGHT_PRED, VERT_RIGHT_PRED, HOR_DOWN_PRED, VERT_LEFT_PRED, HOR_UP_PRED,
 TM_VP8_PRED, LEFT_DC_PRED, TOP_DC_PRED, DC_128_PRED, DC_127_PRED, DC_129_PRED) = range(15)    # IntraPredMode, libavcodec/vp9.h:45-61
INTRA_HAVE_LEFT, INTRA_HAVE_RIGHT, INTRA_LOSSLESS = 1, 2, 4            # B200Vp9IntraOp.flags
INTRA_DTYPE = np.dtype([("coef_off", "<i8"), ("x", "<i4"), ("y", "<i4"), ("eob", "<u2"), ("plane", "u1"), ("tx", "u1"), ("mode", "u1"),
                        ("flags", "u1"), ("reserved", "u1", 10)])
assert INTRA_DTYPE.itemsize == C.sizeof(Vp9IntraOp) == 32


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_vp9dsp_init(bit_depth=8):
    """VP9DSPContext with mc[5][4][2][2][2] and smc[5][4][2] filled (HOST pointers), every other member NULL"""
    c = VP9DSPContext()
    check(lib().b200_vp9_dsp_init(C.byref(c), bit_depth), "ff_vp9dsp_init")
    return c


def vp9_mc_batch_device(device, bit_depth, refs, nops, ops, dst, dst_stride):
    """one plane's inter blocks; refs = up to 8 (plane, stride, w, h, dx, dy) with plane a sample tensor or device address of sample
    (0, 0), stride in bytes, steps in sixteenths (16, 16 = same size as the current picture); ops = OP_DTYPE records (a uint8 tensor of
    nops * 40 bytes); dst a sample tensor, dst_stride in bytes (device)"""
    arr = (Vp9McRef * max(1, len(refs)))()
    for k, (plane, stride, w, h, dx, dy) in enumerate(refs):
        arr[k] = Vp9McRef(_dptr(plane), stride, w, h, dx, dy)
    return check(lib().b200_vp9_mc_batch_device(device.handle, bit_depth, len(refs), C.cast(arr, vp), nops, vp(_dptr(ops)), vp(_dptr(dst)),
                                                dst_stride), "vp9_mc_batch_device")


def ff_vp9dsp_init_itxfm(ctx, bit_depth=8):
    """fills ctx.itxfm_add (HOST pointers, plain addresses in the VP9DSPContext mirror: call one through
    VP9_ITXFM_FUNC(ctx.itxfm_add[tx][type])) and touches no other member; returns ctx"""
    check(lib().b200_vp9_dsp_init_itxfm(C.byref(ctx), bit_depth), "ff_vp9dsp_init_itxfm")
    return ctx


def vp9_itxfm_add_batch_device(device, bit_depth, nops, ops, coef, dst, dst_stride):
    """one plane's transform blocks: ops = TX_DTYPE records (a uint8 tensor of nops * 24 bytes), coef = int16 (8 bit) / int32 (10 / 12
    bit) coefficients, read only; dst a sample tensor, dst_stride in bytes (device)"""
    return check(lib().b200_vp9_itxfm_add_batch_device(device.handle, bit_depth, nops, vp(_dptr(ops)), vp(_dptr(coef)), vp(_dptr(dst)),
                                                       dst_stride), "vp9_itxfm_add_batch_device")


def ff_vp9dsp_init_loopfilter(ctx, bit_depth=8):
    """fills ctx.loop_filter_8, loop_filter_16 and loop_filter_mix2 (HOST pointers: call one through VP9_LF_FUNC(ctx.loop_filter_8[wd][dir]))
    and touches no other member; returns ctx"""
    check(lib().b200_vp9_dsp_init_loopfilter(C.byref(ctx), bit_depth), "ff_vp9dsp_init_loopfilter")
    return ctx


def vp9_loopfilter_frame_device(device, bit_depth, ss_h, ss_v, width, height, planes, ls_y, ls_uv, lflvl, lflvl_stride, lim_lut, mblim_lut):
    """the whole frame's loop filter in place: planes = 3 sample tensors (or device addresses), line sizes in bytes; lflvl = LF_DTYPE records
    (a uint8 tensor), lflvl_stride records per superblock row; lim_lut / mblim_lut = 64 host bytes each (the decoder's filter_lut)"""
    arr = (C.c_void_p * 3)(*[_dptr(p) for p in planes])
    lim = (C.c_uint8 * 64)(*[int(v) for v in lim_lut])
    mblim = (C.c_uint8 * 64)(*[int(v) for v in mblim_lut])
    return check(lib().b200_vp9_loopfilter_frame_device(device.handle, bit_depth, ss_h, ss_v, width, height, arr, ls_y, ls_uv, vp(_dptr(lflvl)),
                                                        lflvl_stride, lim, mblim), "vp9_loopfilter_frame_device")


def vp9_loopfilter_timeouts(device):
    """waits of the frame entry that ran out on this device since the process started (after the device's stream is done)"""
    n = C.c_int64()
    check(lib().b200_vp9_loopfilter_timeouts(device.handle, C.byref(n)), "vp9_loopfilter_timeouts")
    return n.value


def ff_vp9dsp_init_intrapred(ctx, bit_depth=8):
    """fills ctx.intra_pred (HOST pointers: call one through VP9_INTRA_FUNC(ctx.intra_pred[tx][mode])) and touches no other member;
    returns ctx"""
    check(lib().b200_vp9_dsp_init_intrapred(C.byref(ctx), bit_depth), "ff_vp9dsp_init_intrapred")
    return ctx


def vp9_intra_recon_frame_device(device, bit_depth, ss_h, ss_v, width, height, planes, ls_y, ls_uv, nops, ops, coef):
    """every intra transform block of a frame in decode order, in place: planes = 3 sample tensors (or device addresses), line sizes in
    bytes; ops = INTRA_DTYPE records (a uint8 tensor of nops * 32 bytes); coef = int16 (8 bit) / int32 (10 / 12 bit) coefficients, read
    only (device)"""
    arr = (C.c_void_p * 3)(*[_dptr(p) for p in planes])
    return check(lib().b200_vp9_intra_recon_frame_device(device.handle, bit_depth, ss_h, ss_v, width, height, arr, ls_y, ls_uv, nops,
                                                         vp(_dptr(ops)), vp(_dptr(coef))), "vp9_intra_recon_frame_device")


def vp9_intra_timeouts(device):
    """waits of the intra frame entry that ran out on this device since the process started (after the device's stream is done)"""
    n = C.c_int64()
    check(lib().b200_vp9_intra_timeouts(device.handle, C.byref(n)), "vp9_intra_timeouts")
    return n.value
