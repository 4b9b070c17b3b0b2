"""Host-side mirror of libavcodec's HEVC DSP: the put_hevc_{q,e}pel tables of HEVCDSPContext as ff_hevc_dsp_init installs them
(libavcodec/hevc/dsp.c:140-196) and the batched device entry b200_hevc_mc_batch_device; the residual members (hevc/dsp.c:198-215) and
the batched device entry b200_hevc_transform_add_batch_device; the loop-filter members (hevc/dsp.c:237-244) and the plane entry
b200_hevc_deblock_plane_device; the sample adaptive offset members (hevc/dsp.c:217-228) and the out-of-place plane entry
b200_hevc_sao_plane_device; HEVCPredContext (hevc/pred.c) and the batched intra prediction entry b200_hevc_intra_pred_batch_device."""
import ctypes as C

import numpy as np

from ._lib import lib, check, vp, HEVCDSPContext, HevcMcOp, HevcTuOp, HevcDbkSeg, HevcSaoCtb, SAOParams, HevcIntraOp, HEVCPredContext, \
    HevcIntraReconOp

UNI, UNI_W, BI, BI_W = range(4)                 # B200HevcMcOp.kind
OP_DTYPE = np.dtype([("dst_off", "<i8"), ("ref_off", "<i8", 2), ("x", "<i4", 2), ("y", "<i4", 2), ("mx", "u1", 2), ("my", "u1", 2),
                     ("w", "u1"), ("h", "u1"), ("kind", "u1"), ("denom", "u1"), ("wx0", "<i4"), ("wx1", "<i4"), ("ox", "<i4"),
                     ("reserved", "u1", 4)])
assert OP_DTYPE.itemsize == C.sizeof(HevcMcOp) == 64

IDCT, IDCT_DC, DST4, SKIP, BYPASS = range(5)    # B200HevcTuOp.kind
RDPCM, RDPCM_VER, ROTATE = 1, 2, 4              # B200HevcTuOp.flags
TU_DTYPE = np.dtype([("dst_off", "<i8"), ("coef_off", "<i8"), ("log2_size", "u1"), ("kind", "u1"), ("flags", "u1"), ("reserved0", "u1"),
                     ("col_limit", "<i4"), ("reserved", "u1", 8)])
assert TU_DTYPE.itemsize == C.sizeof(HevcTuOp) == 32

# the residual members' signatures (HEVCDSPContext keeps them as plain pointers; cast with these to call one)
ADD_RESIDUAL = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)
DEQUANT = C.CFUNCTYPE(None, C.c_void_p, C.c_int16)
TRANSFORM_RDPCM = C.CFUNCTYPE(None, C.c_void_p, C.c_int16, C.c_int)
TRANSFORM_4X4_LUMA = C.CFUNCTYPE(None, C.c_void_p)
IDCT_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int)
IDCT_DC_FN = C.CFUNCTYPE(None, C.c_void_p)

NO_P, NO_Q = 1, 2                               # B200HevcDbkSeg.flags
DBK_DTYPE = np.dtype([("beta", "u1"), ("tc", "u1"), ("flags", "u1"), ("reserved", "u1")])
assert DBK_DTYPE.itemsize == C.sizeof(HevcDbkSeg) == 4

# the loop-filter members' signatures: (pix, stride, beta, tc[2], no_p[2], no_q[2]) for luma, (pix, stride, tc[2], no_p[2], no_q[2]) for
# chroma
LOOP_FILTER_LUMA = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p)
LOOP_FILTER_CHROMA = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_void_p, C.c_void_p)

SAO_NONE, SAO_BAND, SAO_EDGE = range(3)         # B200HevcSaoCtb.type
(SAO_RESTORE, SAO_VERT_L, SAO_VERT_R, SAO_HORIZ_T, SAO_HORIZ_B, SAO_DIAG_TL, SAO_DIAG_TR, SAO_DIAG_BR,
 SAO_DIAG_BL) = (1 << k for k in range(9))      # B200HevcSaoCtb.flags
SAO_DTYPE = np.dtype([("offset_val", "<i2", 5), ("type", "u1"), ("cls", "u1"), ("flags", "<u2"), ("reserved", "<u2")])
assert SAO_DTYPE.itemsize == C.sizeof(HevcSaoCtb) == 16
assert C.sizeof(SAOParams) == 148

# the SAO members' signatures: band (dst, src, stride_dst, stride_src, offset_val, left_class, width, height); edge (dst, src at the
# 192-byte stride, stride_dst, offset_val, eo_class, width, height); restore (dst, src, stride_dst, stride_src, sao, borders, width,
# height, c_idx, vert_edge, horiz_edge, diag_edge)
SAO_BAND_FILTER = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_int, C.c_int, C.c_int)
SAO_EDGE_FILTER = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_int, C.c_int, C.c_int)
SAO_EDGE_RESTORE = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                               C.c_void_p, C.c_void_p, C.c_void_p)

(INTRA_CAND_BL, INTRA_CAND_L, INTRA_CAND_UL, INTRA_CAND_U, INTRA_CAND_UR, INTRA_LUMA, INTRA_SMOOTH,
 INTRA_STRONG) = (1 << k for k in range(8))     # B200HevcIntraOp.flags
INTRA_DTYPE = np.dtype([("x", "<i4"), ("y", "<i4"), ("log2_size", "u1"), ("mode", "u1"), ("flags", "<u2"), ("reserved", "u1", 4)])
assert INTRA_DTYPE.itemsize == C.sizeof(HevcIntraOp) == 16

TU_NONE = 0xFF                                  # B200HevcIntraReconOp.tu_kind of a TU without residual (cbf 0)
RECON_DTYPE = np.dtype([("coef_off", "<i8"), ("x", "<i4"), ("y", "<i4"), ("plane", "u1"), ("log2_size", "u1"), ("mode", "u1"),
                        ("tu_kind", "u1"), ("flags", "<u2"), ("tu_flags", "u1"), ("reserved0", "u1"), ("col_limit", "<i4"),
                        ("reserved", "u1", 4)])
assert RECON_DTYPE.itemsize == C.sizeof(HevcIntraReconOp) == 32

# HEVCPredContext's member signatures: planar (src, top, left, stride); dc (src, top, left, stride, log2_size, c_idx); angular (src,
# top, left, stride, c_idx, mode); 3-tap (filtered_left, filtered_top, left, top, size); strong (filtered_top, left, top)
PRED_PLANAR = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t)
PRED_DC = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int)
PRED_ANGULAR = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int)
REF_FILTER_3TAP = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int)
REF_FILTER_STRONG = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p)


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_hevc_dsp_init(bit_depth=8):
    """HEVCDSPContext with the six inter-prediction tables filled (HOST pointers), every other member NULL"""
    c = HEVCDSPContext()
    check(lib().b200_hevc_dsp_init(C.byref(c), bit_depth), "ff_hevc_dsp_init")
    return c


def ff_hevc_dsp_init_transform(c, bit_depth=8):
    """fills the residual members of the HEVCDSPContext `c` (HOST pointers: add_residual, dequant, transform_rdpcm,
    transform_4x4_luma, idct, idct_dc), leaving every other member as it is; returns c"""
    check(lib().b200_hevc_dsp_init_transform(C.byref(c), bit_depth), "ff_hevc_dsp_init_transform")
    return c


def hevc_transform_add_batch_device(device, bit_depth, nops, ops, coef, dst, dst_stride):
    """one plane's transform units; ops = TU_DTYPE records (a uint8 tensor of nops * 32 bytes), coef an int16 tensor (not written),
    dst a sample tensor, dst_stride in bytes (device)"""
    return check(lib().b200_hevc_transform_add_batch_device(device.handle, bit_depth, nops, vp(_dptr(ops)), vp(_dptr(coef)), vp(_dptr(dst)),
                                                            dst_stride), "hevc_transform_add_batch_device")


def ff_hevc_dsp_init_deblock(c, bit_depth=8):
    """fills the eight loop-filter members of the HEVCDSPContext `c` (HOST pointers; each _c member equal to its plain twin), leaving
    every other member as it is; returns c"""
    check(lib().b200_hevc_dsp_init_deblock(C.byref(c), bit_depth), "ff_hevc_dsp_init_deblock")
    return c


def hevc_deblock_plane_device(device, bit_depth, chroma, pix, stride, width, height, vseg, vseg_stride, hseg, hseg_stride):
    """deblocks one plane in place (device); pix a sample tensor, stride in bytes; vseg / hseg DBK_DTYPE grids (uint8 tensors of 4-byte
    records) with their strides in records"""
    return check(lib().b200_hevc_deblock_plane_device(device.handle, bit_depth, chroma, vp(_dptr(pix)), stride, width, height, vp(_dptr(vseg)),
                                                      vseg_stride, vp(_dptr(hseg)), hseg_stride), "hevc_deblock_plane_device")


def ff_hevc_dsp_init_sao(c, bit_depth=8):
    """fills the SAO members of the HEVCDSPContext `c` (HOST pointers: sao_band_filter[5], sao_edge_filter[5], sao_edge_restore[2]),
    leaving every other member as it is; returns c"""
    check(lib().b200_hevc_dsp_init_sao(C.byref(c), bit_depth), "ff_hevc_dsp_init_sao")
    return c


def hevc_sao_plane_device(device, bit_depth, dst, dst_stride, src, src_stride, width, height, log2_ctb_size, hshift, vshift, ctb, ctb_stride,
                          keep=None, keep_stride=0, log2_min_pu_size=0):
    """applies SAO to one plane out of place (device): dst / src sample tensors (not overlapping), strides in bytes; ctb a SAO_DTYPE
    grid (a uint8 tensor of 16-byte records) with its stride in records; keep None or the is_pcm map (uint8, one byte per luma min PU)"""
    return check(lib().b200_hevc_sao_plane_device(device.handle, bit_depth, vp(_dptr(dst)), dst_stride, vp(_dptr(src)), src_stride, width,
                                                  height, log2_ctb_size, hshift, vshift, vp(_dptr(ctb)), ctb_stride,
                                                  None if keep is None else vp(_dptr(keep)), keep_stride, log2_min_pu_size),
                 "hevc_sao_plane_device")


def ff_hevc_pred_init(bit_depth=8):
    """a HEVCPredContext with every member ff_hevc_pred_init fills except intra_pred[] (NULL): HOST pointers"""
    c = HEVCPredContext()
    check(lib().b200_hevc_pred_init(C.byref(c), bit_depth), "ff_hevc_pred_init")
    return c


def hevc_intra_pred_batch_device(device, bit_depth, pix, stride, width, height, hshift, vshift, nops, ops, intra_map=None, map_stride=0,
                                 log2_min_pu_size=0):
    """one call of independent intra TUs on one plane (device): pix a sample tensor, stride in bytes, width / height the LUMA picture
    size; ops = INTRA_DTYPE records (a uint8 tensor of nops * 16 bytes); intra_map None (constrained_intra_pred_flag 0) or a uint8
    tensor, one byte per luma min PU"""
    return check(lib().b200_hevc_intra_pred_batch_device(device.handle, bit_depth, vp(_dptr(pix)), stride, width, height, hshift, vshift, nops,
                                                         vp(_dptr(ops)), None if intra_map is None else vp(_dptr(intra_map)), map_stride,
                                                         log2_min_pu_size), "hevc_intra_pred_batch_device")


def hevc_intra_recon_picture_device(device, bit_depth, chroma_format_idc, width, height, planes, ls_y, ls_uv, nops, ops, coef,
                                    intra_map=None, map_stride=0, log2_min_pu_size=0):
    """every intra TU of a picture, all components, in decode order, in place (device): planes = 3 sample tensors (or device addresses;
    only the first with chroma_format_idc 0), line sizes in bytes; ops = RECON_DTYPE records (a uint8 tensor of nops * 32 bytes); coef
    an int16 tensor, read only; intra_map as for hevc_intra_pred_batch_device"""
    arr = (C.c_void_p * 3)(*[_dptr(p) if p is not None else None for p in (list(planes) + [None, None])[:3]])
    return check(lib().b200_hevc_intra_recon_picture_device(device.handle, bit_depth, chroma_format_idc, width, height, arr, ls_y, ls_uv, nops,
                                                            vp(_dptr(ops)), vp(_dptr(coef)),
                                                            None if intra_map is None else vp(_dptr(intra_map)), map_stride,
                                                            log2_min_pu_size), "hevc_intra_recon_picture_device")


def hevc_intra_timeouts(device):
    """waits of the intra picture entry that ran out on this device since the process started (after the device's stream is done)"""
    n = C.c_int64()
    check(lib().b200_hevc_intra_timeouts(device.handle, C.byref(n)), "hevc_intra_timeouts")
    return n.value


def hevc_mc_batch_device(device, bit_depth, epel, nops, ops, dst, dst_stride, ref, ref_stride, pic_w, pic_h):
    """one plane's prediction units; ops = OP_DTYPE records (a uint8 tensor of nops * 64 bytes), dst / ref sample tensors, strides in
    bytes (device)"""
    return check(lib().b200_hevc_mc_batch_device(device.handle, bit_depth, epel, nops, vp(_dptr(ops)), vp(_dptr(dst)), dst_stride,
                                                 vp(_dptr(ref)), ref_stride, pic_w, pic_h), "hevc_mc_batch_device")
