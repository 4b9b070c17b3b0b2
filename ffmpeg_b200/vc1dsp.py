"""Host-side mirror of libavcodec's VC-1 / WMV3 DSP: the transforms and MC tables of VC1DSPContext as ff_vc1dsp_init installs them
(libavcodec/vc1dsp.c:968-1017; overlap, loop filter, sprite and start-code members left NULL), and the two one-call-per-frame device
entries: b200_vc1_mc_frame_device (ff_vc1_mc_1mv / ff_vc1_mc_4mv_luma / ff_vc1_mc_4mv_chroma / ff_vc1_interp_mc over every inter block of a
progressive picture, vc1_mc.c:172-836, :1004-1230) and b200_vc1_residual_frame_device (vc1_decode_p_block's transform calls over every
inter 8x8 block, vc1_block.c:1124-1240)."""
import ctypes as C

import numpy as np

from ._lib import lib, check, vp, VC1DSPContext, Vc1McRef, Vc1McSrc, Vc1McOp, Vc1ResidualOp  # noqa: F401

MC_1MV, MC_LUMA8, MC_CHROMA8 = range(3)                               # B200Vc1McOp.kind
MSPEL, RND, AVG = 1, 2, 4                                             # B200Vc1McOp.flags
TT_8X8, TT_8X4, TT_4X8, TT_4X4 = range(4)                             # B200Vc1ResidualOp.ttblk
MAX_REFS = 2
SRC_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("uvx", "<i2"), ("uvy", "<i2"), ("ref", "u1"), ("mx", "u1"), ("my", "u1"), ("uvmx", "u1"),
                      ("uvmy", "u1"), ("reserved", "u1", 3)])
MC_DTYPE = np.dtype([("dst_x", "<i2"), ("dst_y", "<i2"), ("kind", "u1"), ("flags", "u1"), ("reserved", "u1", 2), ("src", SRC_DTYPE, (2,))])
assert SRC_DTYPE.itemsize == C.sizeof(Vc1McSrc) == 16 and MC_DTYPE.itemsize == C.sizeof(Vc1McOp) == 40
RES_DTYPE = np.dtype([("coef_off", "<i8"), ("x", "<i2"), ("y", "<i2"), ("plane", "u1"), ("ttblk", "u1"), ("subblkpat", "u1"), ("dc", "u1")])
assert RES_DTYPE.itemsize == C.sizeof(Vc1ResidualOp) == 16


class VC1RefDesc:
    """one reference picture of vc1_mc_frame_device: planes (uint8 tensors or device addresses of sample (0, 0)), line sizes in bytes,
    rangeredfrm, use_ic with luty / lutuv ([2][256] uint8, indexed by source-row parity), interlaced (refused by the entry)"""

    def __init__(self, y, u, v, ls_y, ls_uv, rangeredfrm=0, use_ic=0, luty=None, lutuv=None, interlaced=0):
        self.y, self.u, self.v, self.ls_y, self.ls_uv = y, u, v, ls_y, ls_uv
        self.rangeredfrm, self.use_ic, self.interlaced = rangeredfrm, use_ic, interlaced
        ident = np.tile(np.arange(256, dtype=np.uint8), (2, 1))
        self.luty = np.ascontiguousarray(ident if luty is None else luty, np.uint8)
        self.lutuv = np.ascontiguousarray(ident if lutuv is None else lutuv, np.uint8)

    def struct(self, ptr=None):
        """the B200Vc1McRef; `ptr` maps a plane to its address (default: data_ptr() of a tensor, or the int itself)"""
        ptr = ptr or _dptr
        r = Vc1McRef(ptr(self.y), ptr(self.u), ptr(self.v), self.ls_y, self.ls_uv, int(self.rangeredfrm), int(self.use_ic), int(self.interlaced), 0)
        C.memmove(r.luty, self.luty.ctypes.data, 512)
        C.memmove(r.lutuv, self.lutuv.ctypes.data, 512)
        return r


def ref_array(refs, ptr=None):
    arr = (Vc1McRef * max(1, len(refs)))()
    for k, r in enumerate(refs):
        arr[k] = r.struct(ptr)
    return arr


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_vc1dsp_init():
    """VC1DSPContext with the transforms and MC tables filled (HOST pointers), every other member NULL"""
    c = VC1DSPContext()
    check(lib().b200_vc1_dsp_init(C.byref(c)), "ff_vc1dsp_init")
    return c


def vc1_mc_frame_device(device, refs, dst, ls_y, ls_uv, mb_width, mb_height, h_edge_pos, v_edge_pos, nops, ops):
    """every inter block of a progressive picture: refs = up to 2 VC1RefDesc; dst = the 3 planes written (device), line sizes in bytes;
    ops = MC_DTYPE records (a uint8 tensor of nops * 40 bytes, or a device address)"""
    arr = ref_array(refs)
    planes = (C.c_void_p * 3)(*[_dptr(p) for p in dst])
    return check(lib().b200_vc1_mc_frame_device(device.handle, len(refs), C.cast(arr, vp), planes, ls_y, ls_uv, mb_width, mb_height, h_edge_pos,
                                                v_edge_pos, nops, vp(_dptr(ops))), "vc1_mc_frame_device")


def vc1_residual_frame_device(device, dst, ls_y, ls_uv, mb_width, mb_height, coef, nops, ops):
    """every inter 8x8 block's transforms: dst = the 3 planes, updated in place (device), line sizes in bytes; coef = int16 coefficients,
    64 per block in raster order, read only; ops = RES_DTYPE records (a uint8 tensor of nops * 16 bytes, or a device address)"""
    planes = (C.c_void_p * 3)(*[_dptr(p) for p in dst])
    return check(lib().b200_vc1_residual_frame_device(device.handle, planes, ls_y, ls_uv, mb_width, mb_height, vp(_dptr(coef)), nops,
                                                      vp(_dptr(ops))), "vc1_residual_frame_device")
