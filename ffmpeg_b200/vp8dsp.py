"""Host-side mirror of libavcodec's VP8 / VP7 DSP: the MC tables and the six residual members of VP8DSPContext as ff_vp78dsp_init plus
ff_vp8dsp_init / ff_vp7dsp_init install them (libavcodec/vp8dsp.c:641-760; ff_vp8dsp_init leaves the loop-filter members NULL), the
ten loop-filter members (ff_vp8dsp_init_loopfilter, vp8dsp.c:263-457), and the three one-call-per-frame device entries:
b200_vp8_mc_frame_device (vp8_mc_luma / vp8_mc_chroma over every inter block, vp8.c:1831-2083), b200_vp8_residual_frame_device (the
luma DC WHT and idct_mb over every macroblock, vp8.c:1517-1524, :2085-2146) and b200_vp8_loopfilter_frame_device (filter_mb_row over
every macroblock row, vp8.c:2523-2574)."""
import ctypes as C

import numpy as np

from ._lib import (lib, check, vp, VP8DSPContext, Vp8McRef, Vp8McOp, Vp8ResidualOp, Vp8FilterStrength, VP8_MC_FUNC, VP8_WHT_FUNC,  # noqa: F401
                   VP8_IDCT_FUNC, VP8_LF_FUNC, VP8_LF_UV_FUNC, VP8_LF_SIMPLE_FUNC)

LUMA, CHROMA = range(2)                                               # B200Vp8McOp.plane
RESIDUAL_LUMA = 1                                                     # B200Vp8ResidualOp.flags
MAX_REFS = 3
MC_DTYPE = np.dtype([("src_x", "<i4"), ("src_y", "<i4"), ("dst_x", "<i4"), ("dst_y", "<i4"), ("plane", "u1"), ("w", "u1"), ("h", "u1"),
                     ("ref", "u1"), ("mx", "u1"), ("my", "u1"), ("reserved", "u1", 2)])
assert MC_DTYPE.itemsize == C.sizeof(Vp8McOp) == 24
RES_DTYPE = np.dtype([("coef_off", "<i8"), ("mb_x", "<i4"), ("mb_y", "<i4"), ("nnz", "u1", (6, 4)), ("y2_nnz", "u1"), ("flags", "u1"),
                      ("reserved", "u1", 6)])
assert RES_DTYPE.itemsize == C.sizeof(Vp8ResidualOp) == 48
MB_COEFS = 400                                                        # td->block[6][4][16], then block_dc[16]
LF_DTYPE = np.dtype([("filter_level", "u1"), ("inner_limit", "u1"), ("inner_filter", "u1")])
assert LF_DTYPE.itemsize == C.sizeof(Vp8FilterStrength) == 3


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_vp8dsp_init(is_vp7=0):
    """VP8DSPContext with the MC tables and the residual members filled (HOST pointers), the loop-filter members NULL"""
    c = VP8DSPContext()
    check(lib().b200_vp8_dsp_init(C.byref(c), is_vp7), "ff_vp8dsp_init")
    return c


def vp8_mc_frame_device(device, bilinear, mb_width, mb_height, refs, nops, ops, dst, ls_y, ls_uv):
    """every inter block of a frame: refs = up to 3 (y, u, v, ls_y, ls_uv) with planes as uint8 tensors or device addresses of sample
    (0, 0); ops = MC_DTYPE records (a uint8 tensor of nops * 24 bytes); dst = the 3 planes written (device), line sizes in bytes"""
    arr = (Vp8McRef * max(1, len(refs)))()
    for k, (y, u, v, rls_y, rls_uv) in enumerate(refs):
        arr[k] = Vp8McRef(_dptr(y), _dptr(u), _dptr(v), rls_y, rls_uv)
    planes = (C.c_void_p * 3)(*[_dptr(p) for p in dst])
    return check(lib().b200_vp8_mc_frame_device(device.handle, int(bool(bilinear)), mb_width, mb_height, len(refs), C.cast(arr, vp), nops,
                                                vp(_dptr(ops)), planes, ls_y, ls_uv), "vp8_mc_frame_device")


def vp8_residual_frame_device(device, is_vp7, nops, ops, coef, dst, ls_y, ls_uv):
    """every macroblock's residual: ops = RES_DTYPE records (a uint8 tensor of nops * 48 bytes); coef = int16 coefficients, MB_COEFS per
    macroblock, read only; dst = the 3 planes, updated in place (device), line sizes in bytes"""
    planes = (C.c_void_p * 3)(*[_dptr(p) for p in dst])
    return check(lib().b200_vp8_residual_frame_device(device.handle, is_vp7, nops, vp(_dptr(ops)), vp(_dptr(coef)), planes, ls_y, ls_uv),
                 "vp8_residual_frame_device")


def ff_vp8dsp_init_loopfilter(ctx, is_vp7=0):
    """fills the ten loop-filter members of ctx (HOST pointers: call them through ctx.vp8_v_loop_filter16y(...) and so on) and touches
    no other member; returns ctx"""
    check(lib().b200_vp8_dsp_init_loopfilter(C.byref(ctx), is_vp7), "ff_vp8dsp_init_loopfilter")
    return ctx


def vp8_loopfilter_frame_device(device, is_vp7, simple, keyframe, mb_width, mb_height, planes, ls_y, ls_uv, f, f_stride):
    """the whole frame's loop filter in place: planes = 3 uint8 tensors (or device addresses), line sizes in bytes; f = LF_DTYPE records
    (a uint8 tensor or a device address, any byte alignment), f[mb_y * f_stride + mb_x]"""
    arr = (C.c_void_p * 3)(*[_dptr(p) for p in planes])
    return check(lib().b200_vp8_loopfilter_frame_device(device.handle, is_vp7, simple, keyframe, mb_width, mb_height, arr, ls_y, ls_uv,
                                                        vp(_dptr(f)), f_stride), "vp8_loopfilter_frame_device")


def vp8_loopfilter_timeouts(device):
    """waits of the loop-filter frame entry that ran out on this device since the process started (after the device's stream is done)"""
    n = C.c_int64()
    check(lib().b200_vp8_loopfilter_timeouts(device.handle, C.byref(n)), "vp8_loopfilter_timeouts")
    return n.value
