"""ctypes binding of libb200dsp.so (the C ABI declared in include/b200dsp.h).

The library is built in-tree by `__graft_entry__.build()` (ffmpeg_b200/csrc/Makefile, nvcc, sm_90a only).
There is no fallback: if the shared object is missing, or no CUDA device is usable, everything here raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libb200dsp.so")

u8p = C.POINTER(C.c_uint8)
i16p = C.POINTER(C.c_int16)
i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
vp = C.c_void_p


class B200Error(RuntimeError):
    pass


class IDCTDSPContext(C.Structure):
    """Same member order as IDCTDSPContext, libavcodec/idctdsp.h:43-91."""
    _fields_ = [
        ("put_pixels_clamped", C.CFUNCTYPE(None, i16p, u8p, C.c_ssize_t)),
        ("put_signed_pixels_clamped", C.CFUNCTYPE(None, i16p, u8p, C.c_ssize_t)),
        ("add_pixels_clamped", C.CFUNCTYPE(None, i16p, u8p, C.c_ssize_t)),
        ("idct", C.CFUNCTYPE(None, i16p)),
        ("idct_put", C.CFUNCTYPE(None, u8p, C.c_ssize_t, i16p)),
        ("idct_add", C.CFUNCTYPE(None, u8p, C.c_ssize_t, i16p)),
        ("idct_permutation", C.c_uint8 * 64),
        ("perm_type", C.c_int),
        ("mpeg4_studio_profile", C.c_int),
    ]


_CMP = C.CFUNCTYPE(C.c_int, C.c_void_p, u8p, u8p, C.c_ssize_t, C.c_int)


class MECmpContext(C.Structure):
    """Same member order as MECmpContext, libavcodec/me_cmp.h:53-77."""
    _fields_ = [("sum_abs_dctelem", C.CFUNCTYPE(C.c_int, i16p))] + \
        [(n, _CMP * 6) for n in ("sad", "sse", "hadamard8_diff", "dct_sad", "quant_psnr", "bit", "rd", "vsad", "vsse",
                                 "nsse", "w53", "w97", "dct_max", "dct264_sad")] + \
        [("pix_abs", (_CMP * 4) * 2), ("median_sad", _CMP * 6)]


class FDCTDSPContext(C.Structure):
    """Same member order as FDCTDSPContext, libavcodec/fdctdsp.h:28-31."""
    _fields_ = [("fdct", C.CFUNCTYPE(None, i16p)), ("fdct248", C.CFUNCTYPE(None, i16p))]


_QPEL = C.CFUNCTYPE(None, u8p, u8p, C.c_ssize_t)
_HPEL = C.CFUNCTYPE(None, u8p, u8p, C.c_ssize_t, C.c_int)


class H264QpelContext(C.Structure):
    """libavcodec/h264qpel.h:27-30"""
    _fields_ = [("put_h264_qpel_pixels_tab", (_QPEL * 16) * 3), ("avg_h264_qpel_pixels_tab", (_QPEL * 16) * 3)]


class HpelDSPContext(C.Structure):
    """libavcodec/hpeldsp.h:39-97"""
    _fields_ = [("put_pixels_tab", (_HPEL * 4) * 4), ("avg_pixels_tab", (_HPEL * 4) * 4),
                ("put_no_rnd_pixels_tab", (_HPEL * 4) * 3), ("avg_no_rnd_pixels_tab", _HPEL * 4)]


_H264IDCT = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)


class SwsVector(C.Structure):
    """SwsVector (libswscale/swscale.h:187-192)"""
    _fields_ = [("coeff", C.POINTER(C.c_double)), ("length", C.c_int)]


class SwsFilter(C.Structure):
    """SwsFilter (libswscale/swscale.h:199-204)"""
    _fields_ = [("lumH", C.POINTER(SwsVector)), ("lumV", C.POINTER(SwsVector)), ("chrH", C.POINTER(SwsVector)), ("chrV", C.POINTER(SwsVector))]


class H264IDCTContext(C.Structure):
    """the IDCT members of H264DSPContext, libavcodec/h264dsp.h:81-88"""
    _fields_ = [("idct_add", _H264IDCT), ("idct8_add", _H264IDCT), ("idct_dc_add", _H264IDCT), ("idct8_dc_add", _H264IDCT)]


_H264W = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int)
_H264BW = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)


class H264WeightContext(C.Structure):
    """weight_pixels_tab / biweight_pixels_tab of H264DSPContext, libavcodec/h264dsp.h:33-45"""
    _fields_ = [("weight_pixels_tab", _H264W * 4), ("biweight_pixels_tab", _H264BW * 4)]


class FloatDSPContext(C.Structure):
    """AVFloatDSPContext, libavutil/float_dsp.h:24-210 (same member order)"""
    _F, _D = C.POINTER(C.c_float), C.POINTER(C.c_double)
    _fields_ = [("vector_fmul", C.CFUNCTYPE(None, _F, _F, _F, C.c_int)),
                ("vector_fmac_scalar", C.CFUNCTYPE(None, _F, _F, C.c_float, C.c_int)),
                ("vector_dmac_scalar", C.CFUNCTYPE(None, _D, _D, C.c_double, C.c_int)),
                ("vector_fmul_scalar", C.CFUNCTYPE(None, _F, _F, C.c_float, C.c_int)),
                ("vector_dmul_scalar", C.CFUNCTYPE(None, _D, _D, C.c_double, C.c_int)),
                ("vector_fmul_window", C.CFUNCTYPE(None, _F, _F, _F, _F, C.c_int)),
                ("vector_fmul_add", C.CFUNCTYPE(None, _F, _F, _F, _F, C.c_int)),
                ("vector_fmul_reverse", C.CFUNCTYPE(None, _F, _F, _F, C.c_int)),
                ("butterflies_float", C.CFUNCTYPE(None, _F, _F, C.c_int)),
                ("scalarproduct_float", C.CFUNCTYPE(C.c_float, _F, _F, C.c_int)),
                ("vector_dmul", C.CFUNCTYPE(None, _D, _D, _D, C.c_int)),
                ("scalarproduct_double", C.CFUNCTYPE(C.c_double, _D, _D, C.c_size_t))]


_LF_TC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p)
_LF_INTRA = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int)


class H264LoopFilterContext(C.Structure):
    """the loop-filter members of H264DSPContext, libavcodec/h264dsp.h:48-73"""
    _fields_ = [("v_loop_filter_luma", _LF_TC), ("h_loop_filter_luma", _LF_TC), ("h_loop_filter_luma_mbaff", _LF_TC),
                ("v_loop_filter_luma_intra", _LF_INTRA), ("h_loop_filter_luma_intra", _LF_INTRA), ("h_loop_filter_luma_mbaff_intra", _LF_INTRA),
                ("v_loop_filter_chroma", _LF_TC), ("h_loop_filter_chroma", _LF_TC), ("h_loop_filter_chroma_mbaff", _LF_TC),
                ("v_loop_filter_chroma_intra", _LF_INTRA), ("h_loop_filter_chroma_intra", _LF_INTRA), ("h_loop_filter_chroma_mbaff_intra", _LF_INTRA)]


_PRED4 = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)
_PRED8L = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_ssize_t)
_PRED = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t)
_PRED_ADD = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)
_PRED_FADD = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_ssize_t)
_PRED_TADD = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t)


class H264PredContext(C.Structure):
    """libavcodec/h264pred.h:94-114 (same member order and table sizes)"""
    _fields_ = [("pred4x4", _PRED4 * 15), ("pred8x8l", _PRED8L * 12), ("pred8x8", _PRED * 11), ("pred16x16", _PRED * 9),
                ("pred4x4_add", _PRED_ADD * 2), ("pred8x8l_add", _PRED_ADD * 2), ("pred8x8l_filter_add", _PRED_FADD * 2),
                ("pred8x8_add", _PRED_TADD * 3), ("pred16x16_add", _PRED_TADD * 3)]


_QP = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_ssize_t, C.c_ssize_t, C.c_int)
_QP_UNI = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_ssize_t, C.c_ssize_t, C.c_int)
_QP_UNI_W = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_ssize_t,
                        C.c_ssize_t, C.c_int)
_QP_BI = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_int, C.c_ssize_t, C.c_ssize_t, C.c_int)
_QP_BI_W = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                       C.c_ssize_t, C.c_ssize_t, C.c_int)


class HEVCDSPContext(C.Structure):
    """libavcodec/hevc/dsp.h:47-125 (same member order; the members this library does not fill are plain pointers here)"""
    _fields_ = ([("put_pcm", vp), ("add_residual", vp * 4), ("dequant", vp), ("transform_rdpcm", vp), ("transform_4x4_luma", vp),
                 ("idct", vp * 4), ("idct_dc", vp * 4), ("sao_band_filter", vp * 5), ("sao_edge_filter", vp * 5), ("sao_edge_restore", vp * 2)] +
                [(f"put_hevc_{p}{s}", t * 2 * 2 * 10) for p in ("qpel", "epel")
                 for s, t in (("", _QP), ("_uni", _QP_UNI), ("_uni_w", _QP_UNI_W), ("_bi", _QP_BI), ("_bi_w", _QP_BI_W))] +
                [(n, vp) for n in ("hevc_h_loop_filter_luma", "hevc_v_loop_filter_luma", "hevc_h_loop_filter_chroma", "hevc_v_loop_filter_chroma",
                                   "hevc_h_loop_filter_luma_c", "hevc_v_loop_filter_luma_c", "hevc_h_loop_filter_chroma_c",
                                   "hevc_v_loop_filter_chroma_c")])


class HevcMcOp(C.Structure):
    """B200HevcMcOp (include/b200dsp.h), 64 bytes"""
    _fields_ = [("dst_off", C.c_int64), ("ref_off", C.c_int64 * 2), ("x", C.c_int32 * 2), ("y", C.c_int32 * 2), ("mx", C.c_uint8 * 2),
                ("my", C.c_uint8 * 2), ("w", C.c_uint8), ("h", C.c_uint8), ("kind", C.c_uint8), ("denom", C.c_uint8), ("wx0", C.c_int32),
                ("wx1", C.c_int32), ("ox", C.c_int32), ("reserved", C.c_uint8 * 4)]


class HevcTuOp(C.Structure):
    """B200HevcTuOp (include/b200dsp.h), 32 bytes"""
    _fields_ = [("dst_off", C.c_int64), ("coef_off", C.c_int64), ("log2_size", C.c_uint8), ("kind", C.c_uint8), ("flags", C.c_uint8),
                ("reserved0", C.c_uint8), ("col_limit", C.c_int32), ("reserved", C.c_uint8 * 8)]


class HevcDbkSeg(C.Structure):
    """B200HevcDbkSeg (include/b200dsp.h), 4 bytes"""
    _fields_ = [("beta", C.c_uint8), ("tc", C.c_uint8), ("flags", C.c_uint8), ("reserved", C.c_uint8)]


class HevcSaoCtb(C.Structure):
    """B200HevcSaoCtb (include/b200dsp.h), 16 bytes"""
    _fields_ = [("offset_val", C.c_int16 * 5), ("type", C.c_uint8), ("cls", C.c_uint8), ("flags", C.c_uint16), ("reserved", C.c_uint16)]


class SAOParams(C.Structure):
    """B200SAOParams = libavcodec/hevc/dsp.h:34-45 SAOParams, 148 bytes"""
    _fields_ = [("offset_abs", (C.c_int32 * 4) * 3), ("offset_sign", (C.c_int32 * 4) * 3), ("band_position", C.c_uint8 * 3),
                ("eo_class", C.c_int32 * 3), ("offset_val", (C.c_int16 * 5) * 3), ("type_idx", C.c_uint8 * 3)]


class HevcIntraOp(C.Structure):
    """B200HevcIntraOp (include/b200dsp.h), 16 bytes"""
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("log2_size", C.c_uint8), ("mode", C.c_uint8), ("flags", C.c_uint16),
                ("reserved", C.c_uint8 * 4)]


class HEVCPredContext(C.Structure):
    """B200HEVCPredContext = libavcodec/hevc/pred.h HEVCPredContext"""
    _fields_ = [("intra_pred", vp * 4), ("pred_planar", vp * 4), ("pred_dc", vp), ("pred_angular", vp * 4), ("ref_filter_3tap", vp * 3),
                ("ref_filter_strong", vp)]


VP9_MC_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)
VP9_SCALED_MC_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)


class VP9DSPContext(C.Structure):
    """libavcodec/vp9dsp.h:40-122 (same member order; the members this library does not fill are plain pointers here)"""
    _fields_ = [("intra_pred", vp * 15 * 4), ("itxfm_add", vp * 4 * 5), ("loop_filter_8", vp * 2 * 3), ("loop_filter_16", vp * 2),
                ("loop_filter_mix2", vp * 2 * 2 * 2), ("mc", VP9_MC_FUNC * 2 * 2 * 2 * 4 * 5), ("smc", VP9_SCALED_MC_FUNC * 2 * 4 * 5)]


class Vp9McRef(C.Structure):
    """B200Vp9McRef (include/b200dsp.h), 32 bytes"""
    _fields_ = [("data", C.c_void_p), ("stride", C.c_ssize_t), ("w", C.c_int32), ("h", C.c_int32), ("dx", C.c_int32), ("dy", C.c_int32)]


class Vp9McOp(C.Structure):
    """B200Vp9McOp (include/b200dsp.h), 40 bytes"""
    _fields_ = [("dst_off", C.c_int64), ("x", C.c_int32 * 2), ("y", C.c_int32 * 2), ("ref", C.c_uint8 * 2), ("mx", C.c_uint8 * 2),
                ("my", C.c_uint8 * 2), ("w", C.c_uint8), ("h", C.c_uint8), ("filter", C.c_uint8), ("kind", C.c_uint8),
                ("reserved", C.c_uint8 * 6)]


VP9_ITXFM_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_int)


class Vp9TxOp(C.Structure):
    """B200Vp9TxOp (include/b200dsp.h), 24 bytes"""
    _fields_ = [("dst_off", C.c_int64), ("coef_off", C.c_int64), ("tx", C.c_uint8), ("type", C.c_uint8), ("eob", C.c_uint16),
                ("reserved", C.c_uint8 * 4)]


VP9_LF_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)


class Vp9Filter(C.Structure):
    """B200Vp9Filter (include/b200dsp.h) = VP9Filter (libavcodec/vp9dec.h:79-83), 192 bytes"""
    _fields_ = [("level", C.c_uint8 * 64), ("mask", C.c_uint8 * 4 * 8 * 2 * 2)]


VP9_INTRA_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_void_p)


class HevcIntraReconOp(C.Structure):
    """B200HevcIntraReconOp (include/b200dsp.h), 32 bytes"""
    _fields_ = [("coef_off", C.c_int64), ("x", C.c_int32), ("y", C.c_int32), ("plane", C.c_uint8), ("log2_size", C.c_uint8), ("mode", C.c_uint8),
                ("tu_kind", C.c_uint8), ("flags", C.c_uint16), ("tu_flags", C.c_uint8), ("reserved0", C.c_uint8), ("col_limit", C.c_int32),
                ("reserved", C.c_uint8 * 4)]


class Vp9IntraOp(C.Structure):
    """B200Vp9IntraOp (include/b200dsp.h), 32 bytes"""
    _fields_ = [("coef_off", C.c_int64), ("x", C.c_int32), ("y", C.c_int32), ("eob", C.c_uint16), ("plane", C.c_uint8), ("tx", C.c_uint8),
                ("mode", C.c_uint8), ("flags", C.c_uint8), ("reserved", C.c_uint8 * 10)]


VP8_MC_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)
VP8_WHT_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p)
VP8_IDCT_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t)
VP8_LF_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)               # 16y, 16y_inner: dst, stride, E, I, H
VP8_LF_UV_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)  # 8uv, 8uv_inner: dstU, dstV, ...
VP8_LF_SIMPLE_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int)                         # simple: dst, stride, flim


class VP8DSPContext(C.Structure):
    """libavcodec/vp8dsp.h:37-82 (same member order and member types)"""
    _fields_ = [("vp8_luma_dc_wht", VP8_WHT_FUNC), ("vp8_luma_dc_wht_dc", VP8_WHT_FUNC), ("vp8_idct_add", VP8_IDCT_FUNC),
                ("vp8_idct_dc_add", VP8_IDCT_FUNC), ("vp8_idct_dc_add4y", VP8_IDCT_FUNC), ("vp8_idct_dc_add4uv", VP8_IDCT_FUNC),
                ("vp8_v_loop_filter16y", VP8_LF_FUNC), ("vp8_h_loop_filter16y", VP8_LF_FUNC),
                ("vp8_v_loop_filter8uv", VP8_LF_UV_FUNC), ("vp8_h_loop_filter8uv", VP8_LF_UV_FUNC),
                ("vp8_v_loop_filter16y_inner", VP8_LF_FUNC), ("vp8_h_loop_filter16y_inner", VP8_LF_FUNC),
                ("vp8_v_loop_filter8uv_inner", VP8_LF_UV_FUNC), ("vp8_h_loop_filter8uv_inner", VP8_LF_UV_FUNC),
                ("vp8_v_loop_filter_simple", VP8_LF_SIMPLE_FUNC), ("vp8_h_loop_filter_simple", VP8_LF_SIMPLE_FUNC),
                ("put_vp8_epel_pixels_tab", VP8_MC_FUNC * 3 * 3 * 3), ("put_vp8_bilinear_pixels_tab", VP8_MC_FUNC * 3 * 3 * 3)]


class Vp8McRef(C.Structure):
    """B200Vp8McRef (include/b200dsp.h), 40 bytes"""
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("ls_y", C.c_ssize_t), ("ls_uv", C.c_ssize_t)]


class Vp8McOp(C.Structure):
    """B200Vp8McOp (include/b200dsp.h), 24 bytes"""
    _fields_ = [("src_x", C.c_int32), ("src_y", C.c_int32), ("dst_x", C.c_int32), ("dst_y", C.c_int32), ("plane", C.c_uint8), ("w", C.c_uint8),
                ("h", C.c_uint8), ("ref", C.c_uint8), ("mx", C.c_uint8), ("my", C.c_uint8), ("reserved", C.c_uint8 * 2)]


class Vp8ResidualOp(C.Structure):
    """B200Vp8ResidualOp (include/b200dsp.h), 48 bytes"""
    _fields_ = [("coef_off", C.c_int64), ("mb_x", C.c_int32), ("mb_y", C.c_int32), ("nnz", C.c_uint8 * 4 * 6), ("y2_nnz", C.c_uint8),
                ("flags", C.c_uint8), ("reserved", C.c_uint8 * 6)]


class Vp8FilterStrength(C.Structure):
    """B200Vp8FilterStrength (include/b200dsp.h) = VP8FilterStrength (libavcodec/vp8.h:90-94), 3 bytes"""
    _fields_ = [("filter_level", C.c_uint8), ("inner_limit", C.c_uint8), ("inner_filter", C.c_uint8)]


VC1_MSPEL_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int)                     # dst, src, stride, rnd
VC1_CHROMA_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)    # dst, src, stride, h, x, y
VC1_ITX8_FUNC = C.CFUNCTYPE(None, C.c_void_p)                                                         # vc1_inv_trans_8x8(block)
VC1_ITX_FUNC = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p)                                 # dest, stride, block


class VC1DSPContext(C.Structure):
    """libavcodec/vc1dsp.h:37-97 (same member order and member types; the members b200_vc1_dsp_init leaves NULL as untyped pointers)"""
    _fields_ = ([("vc1_inv_trans_8x8", VC1_ITX8_FUNC)] +
                [(f"vc1_inv_trans_{n}", VC1_ITX_FUNC) for n in ("8x4", "4x8", "4x4", "8x8_dc", "8x4_dc", "4x8_dc", "4x4_dc")] +
                [(n, C.c_void_p) for n in ("vc1_v_overlap", "vc1_h_overlap", "vc1_v_s_overlap", "vc1_h_s_overlap", "vc1_v_loop_filter4",
                                           "vc1_h_loop_filter4", "vc1_v_loop_filter8", "vc1_h_loop_filter8", "vc1_v_loop_filter16",
                                           "vc1_h_loop_filter16")] +
                [("put_vc1_mspel_pixels_tab", VC1_MSPEL_FUNC * 16 * 2), ("avg_vc1_mspel_pixels_tab", VC1_MSPEL_FUNC * 16 * 2),
                 ("put_no_rnd_vc1_chroma_pixels_tab", VC1_CHROMA_FUNC * 3), ("avg_no_rnd_vc1_chroma_pixels_tab", VC1_CHROMA_FUNC * 3)] +
                [(n, C.c_void_p) for n in ("sprite_h", "sprite_v_single", "sprite_v_double_noscale", "sprite_v_double_onescale",
                                           "sprite_v_double_twoscale", "startcode_find_candidate", "vc1_unescape_buffer")])


class Vc1McRef(C.Structure):
    """B200Vc1McRef (include/b200dsp.h), 1080 bytes"""
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("ls_y", C.c_ssize_t), ("ls_uv", C.c_ssize_t),
                ("rangeredfrm", C.c_int32), ("use_ic", C.c_int32), ("interlaced", C.c_int32), ("reserved", C.c_int32),
                ("luty", C.c_uint8 * 256 * 2), ("lutuv", C.c_uint8 * 256 * 2)]


class Vc1McSrc(C.Structure):
    """B200Vc1McSrc (include/b200dsp.h), 16 bytes"""
    _fields_ = [("x", C.c_int16), ("y", C.c_int16), ("uvx", C.c_int16), ("uvy", C.c_int16), ("ref", C.c_uint8), ("mx", C.c_uint8),
                ("my", C.c_uint8), ("uvmx", C.c_uint8), ("uvmy", C.c_uint8), ("reserved", C.c_uint8 * 3)]


class Vc1McOp(C.Structure):
    """B200Vc1McOp (include/b200dsp.h), 40 bytes"""
    _fields_ = [("dst_x", C.c_int16), ("dst_y", C.c_int16), ("kind", C.c_uint8), ("flags", C.c_uint8), ("reserved", C.c_uint8 * 2),
                ("src", Vc1McSrc * 2)]


class Vc1ResidualOp(C.Structure):
    """B200Vc1ResidualOp (include/b200dsp.h), 16 bytes"""
    _fields_ = [("coef_off", C.c_int64), ("x", C.c_int16), ("y", C.c_int16), ("plane", C.c_uint8), ("ttblk", C.c_uint8),
                ("subblkpat", C.c_uint8), ("dc", C.c_uint8)]


class ProresDSPContext(C.Structure):
    """libavcodec/proresdsp.h:28-35"""
    _fields_ = [("idct_permutation_type", C.c_int), ("idct_permutation", C.c_uint8 * 64),
                ("idct_put", C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_void_p)),
                ("idct_put_bayer", C.c_void_p)]


class MpvUnquant(C.Structure):
    """B200MpvUnquant: the MPVContext fields the inverse quantisers read (libavcodec/mpegvideo.h:70-77,201-203,258)"""
    _fields_ = [("intra_matrix", C.c_uint16 * 64), ("inter_matrix", C.c_uint16 * 64), ("permutated", C.c_uint8 * 64),
                ("raster_end", C.c_uint8 * 64), ("y_dc_scale", C.c_int32), ("c_dc_scale", C.c_int32), ("q_scale_type", C.c_int32),
                ("h263_aic", C.c_int32), ("ac_pred", C.c_int32)]


_CHROMA = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int)


class H264ChromaContext(C.Structure):
    """libavcodec/h264chroma.h:26-31"""
    _fields_ = [("put_h264_chroma_pixels_tab", _CHROMA * 4), ("avg_h264_chroma_pixels_tab", _CHROMA * 4)]


_EDGE = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)
_PREFETCH = C.CFUNCTYPE(None, C.c_void_p, C.c_ssize_t, C.c_int)


class VideoDSPContext(C.Structure):
    """libavcodec/videodsp.h:32-69"""
    _fields_ = [("emulated_edge_mc", _EDGE), ("prefetch", _PREFETCH)]


TX_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t)

# name -> (restype, argtypes): every symbol include/b200dsp.h declares
PROTOTYPES = {
    "b200_abi_version": (C.c_int, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_device_open": (C.c_int, [C.POINTER(vp), C.c_int, vp]),
    "b200_device_close": (None, [vp]),
    "b200_device_sync": (C.c_int, [vp]),
    "b200_device_ordinal": (C.c_int, [vp]),
    "b200_device_stream": (vp, [vp]),
    "b200_device_sm_count": (C.c_int, [vp]),
    "b200_set_default_device": (C.c_int, [vp]),
    "b200_malloc_device": (vp, [vp, C.c_size_t]),
    "b200_free_device": (None, [vp, vp]),
    "b200_malloc_host": (vp, [C.c_size_t]),
    "b200_free_host": (None, [vp]),
    "b200_memcpy_h2d": (C.c_int, [vp, vp, vp, C.c_size_t]),
    "b200_memcpy_d2h": (C.c_int, [vp, vp, vp, C.c_size_t]),
    "b200_launch_count": (C.c_uint64, []),
    "b200_sws_getContext": (vp, [vp] + [C.c_int] * 7),
    "b200_sws_getContext_range": (vp, [vp] + [C.c_int] * 9),
    "b200_sws_getContext_params": (vp, [vp] + [C.c_int] * 9 + [vp]),
    "b200_sws_getContext_filters": (vp, [vp] + [C.c_int] * 9 + [vp, vp, vp]),
    "b200_sws_freeContext": (None, [vp]),
    "b200_sws_setColorspaceDetails": (C.c_int, [vp, i32p, C.c_int, i32p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200_sws_scale": (C.c_int, [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.POINTER(vp), i32p]),
    "b200_sws_func": (C.c_int, [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.POINTER(vp), i32p]),
    "b200_sws_scale_batch_device": (C.c_int, [vp, C.POINTER(vp), i32p, i64p, vp, C.c_int, C.c_int64, C.c_int]),
    "b200_sws_scale_batch_device_planar": (C.c_int, [vp, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.c_int]),
    "b200_sws_scale_batch_host": (C.c_int, [vp, C.POINTER(vp), i32p, i64p, vp, C.c_int, C.c_int64, C.c_int]),
    "b200_sws_info": (C.c_int, [vp, i32p]),
    "b200_sws_get_filter": (C.c_int, [vp, C.c_int, i16p, i32p, C.c_int]),
    "b200_sws_last_path": (C.c_int, [vp]),
    "b200_sws_plan_probe": (C.c_int, [C.c_int] * 6 + [i16p, i32p, C.c_int, i32p]),
    "b200_sws_plan_probe2": (C.c_int, [i32p, i32p, C.c_int, i16p, i32p, C.c_int, i32p]),
    "b200_sws_mma_probe": (C.c_int, [i16p, i32p, C.c_int, C.c_int, i32p, C.c_int, C.POINTER(C.c_uint32), C.c_int, i32p]),
    "b200_idctdsp_init": (C.c_int, [C.POINTER(IDCTDSPContext), C.c_int, C.c_int, C.c_int]),
    "b200_idct_batch_device": (C.c_int, [vp, C.c_int, vp, C.c_int64, vp, vp, vp, C.c_int]),
    "b200_idct_mb420_device": (C.c_int, [vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp), i32p, i64p]),
    "b200_idct_mb420_host": (C.c_int, [vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp), i32p, i64p]),
    "b200_me_cmp_init": (C.c_int, [C.POINTER(MECmpContext), C.c_int]),
    "b200_mpv_unquant_idct_mb420_device": (C.c_int, [vp, C.c_int, vp, C.c_int, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, i32p, i64p]),
    "b200_me_cmp_set_nsse_weight": (None, [C.c_int]),
    "b200_me_cmp_set_dct_algo": (C.c_int, [C.c_int]),
    "b200_sum_abs_dctelem_batch_device": (C.c_int, [vp, vp, C.c_int64, vp]),
    "b200_fdctdsp_init": (C.c_int, [C.POINTER(FDCTDSPContext), C.c_int, C.c_int]),
    "b200_fdct_batch_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int64]),
    "b200_me_cmp_batch_device": (C.c_int, [vp, C.c_int, C.c_int, vp, vp, C.c_ssize_t, C.c_int, vp, vp, C.c_int64, vp]),
    "b200_me_esa_device": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, vp, vp]),
    "b200_h264qpel_init": (C.c_int, [C.POINTER(H264QpelContext), C.c_int]),
    "b200_hpeldsp_init": (C.c_int, [C.POINTER(HpelDSPContext), C.c_int]),
    "b200_h264qpel_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264qpel_hbd_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264_loop_filter_hbd_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, C.c_ssize_t, vp, vp, vp]),
    "b200_h264_idct_hbd_batch_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264_weight_hbd_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264chroma_hbd_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_emulated_edge_mc_hbd_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, C.c_ssize_t, vp, vp, C.c_ssize_t, vp, C.c_int, C.c_int]),
    "b200_hpel_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264_idct_init": (C.c_int, [C.POINTER(H264IDCTContext), C.c_int, C.c_int]),
    "b200_h264_idct_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264_weight_init": (C.c_int, [C.POINTER(H264WeightContext), C.c_int]),
    "b200_h264_weight_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_mpv_unquantize_batch_device": (C.c_int, [vp, C.c_int, vp, vp, C.c_int64, vp, vp, vp]),
    "b200_idctdsp_init_hbd": (C.c_int, [vp, C.c_int, C.c_int, C.c_int]),
    "b200_idct_hbd_batch_device": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_int64, vp, vp, vp, C.c_int]),
    "b200_tx_pfa_tables": (C.c_int, [C.c_int, C.c_int, C.c_float, vp, C.c_int, vp]),
    "b200_tx_dct_table": (C.c_int, [C.c_int, C.c_int, vp, C.c_int]),
    "b200_tx_i32_tables": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_float, vp, C.c_int, vp]),
    "b200_pixelutils_get_sad_fn": (vp, [C.c_int, C.c_int, C.c_int, vp]),
    "b200_pixelutils_sad_batch_device": (C.c_int, [vp, C.c_int, vp, C.c_ssize_t, vp, C.c_ssize_t, vp, vp, C.c_int64, vp]),
    "b200_h264_loop_filter_init": (C.c_int, [vp, C.c_int, C.c_int]),
    "b200_h264_loop_filter_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, vp, C.c_ssize_t, vp, vp, vp]),
    "b200_h264_pred_init": (C.c_int, [vp, C.c_int, C.c_int, C.c_int]),
    "b200_h264_pred_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_h264_pred_add_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_ssize_t, vp, vp]),
    "b200_hevc_dsp_init": (C.c_int, [vp, C.c_int]),
    "b200_hevc_mc_batch_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int64, vp, vp, C.c_ssize_t, vp, C.c_ssize_t, C.c_int, C.c_int]),
    "b200_hevc_dsp_init_transform": (C.c_int, [vp, C.c_int]),
    "b200_hevc_transform_add_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, C.c_ssize_t]),
    "b200_hevc_dsp_init_deblock": (C.c_int, [vp, C.c_int]),
    "b200_hevc_deblock_plane_device": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_ssize_t, C.c_int, C.c_int, vp, C.c_int64, vp, C.c_int64]),
    "b200_hevc_dsp_init_sao": (C.c_int, [vp, C.c_int]),
    "b200_hevc_sao_plane_device": (C.c_int, [vp, C.c_int, vp, C.c_ssize_t, vp, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp,
                                             C.c_int64, vp, C.c_int64, C.c_int]),
    "b200_hevc_pred_init": (C.c_int, [vp, C.c_int]),
    "b200_hevc_intra_pred_batch_device": (C.c_int, [vp, C.c_int, vp, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, vp, vp,
                                                    C.c_ssize_t, C.c_int]),
    "b200_hevc_intra_recon_picture_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_ssize_t, C.c_ssize_t, C.c_int64, vp,
                                                       vp, vp, C.c_ssize_t, C.c_int]),
    "b200_hevc_intra_timeouts": (C.c_int, [vp, vp]),
    "b200_vp9_dsp_init": (C.c_int, [vp, C.c_int]),
    "b200_vp9_mc_batch_device": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_int64, vp, vp, C.c_ssize_t]),
    "b200_vp9_dsp_init_itxfm": (C.c_int, [vp, C.c_int]),
    "b200_vp9_itxfm_add_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, C.c_ssize_t]),
    "b200_vp9_dsp_init_loopfilter": (C.c_int, [vp, C.c_int]),
    "b200_vp9_loopfilter_frame_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_ssize_t, C.c_ssize_t, vp,
                                                   C.c_int64, vp, vp]),
    "b200_vp9_loopfilter_timeouts": (C.c_int, [vp, vp]),
    "b200_vp9_dsp_init_intrapred": (C.c_int, [vp, C.c_int]),
    "b200_vp9_intra_recon_frame_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_ssize_t, C.c_ssize_t, C.c_int64,
                                                    vp, vp]),
    "b200_vp9_intra_timeouts": (C.c_int, [vp, vp]),
    "b200_vp8_dsp_init": (C.c_int, [vp, C.c_int]),
    "b200_vp8_mc_frame_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int64, vp, vp, C.c_ssize_t, C.c_ssize_t]),
    "b200_vp8_residual_frame_device": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, C.c_ssize_t, C.c_ssize_t]),
    "b200_vp8_dsp_init_loopfilter": (C.c_int, [vp, C.c_int]),
    "b200_vp8_loopfilter_frame_device": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_ssize_t, C.c_ssize_t, vp,
                                                   C.c_int64]),
    "b200_vp8_loopfilter_timeouts": (C.c_int, [vp, vp]),
    "b200_vc1_dsp_init": (C.c_int, [vp]),
    "b200_vc1_mc_frame_device": (C.c_int, [vp, C.c_int, vp, vp, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, vp]),
    "b200_vc1_residual_frame_device": (C.c_int, [vp, vp, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, vp, C.c_int64, vp]),
    "b200_proresdsp_init": (C.c_int, [vp, C.c_int]),
    "b200_prores_idct_put_batch_device": (C.c_int, [vp, C.c_int, vp, C.c_int64, vp, vp, vp, vp, C.c_int]),
    "b200_float_dsp_init": (C.c_int, [vp]),
    "b200_float_dsp_batch_device": (C.c_int, [vp, C.c_int, C.c_int64, C.c_int, vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, C.c_double]),
    "b200_videodsp_init": (C.c_int, [C.POINTER(VideoDSPContext), C.c_int]),
    "b200_emulated_edge_mc_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, C.c_ssize_t, vp, vp, C.c_ssize_t, vp, C.c_int, C.c_int]),
    "b200_h264chroma_init": (C.c_int, [C.POINTER(H264ChromaContext), C.c_int]),
    "b200_h264chroma_batch_device": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_tx_init": (C.c_int, [C.POINTER(vp), C.POINTER(TX_FN), C.c_int, C.c_int, C.c_int, vp, C.c_uint64]),
    "b200_tx_init_device": (C.c_int, [vp, C.POINTER(vp), C.POINTER(TX_FN), C.c_int, C.c_int, C.c_int, vp, C.c_uint64]),
    "b200_tx_uninit": (None, [C.POINTER(vp)]),
    "b200_tx_batch_device": (C.c_int, [vp, vp, vp, C.c_ssize_t, C.c_int64, C.c_ssize_t, C.c_ssize_t]),
    "b200_tx_r16_plan": (C.c_int, [C.c_int, C.c_int, vp, C.c_int]),
    "b200_tx_batch_host": (C.c_int, [vp, vp, vp, C.c_ssize_t, C.c_int64, C.c_ssize_t, C.c_ssize_t]),
    "b200_h264qpel_frames_host": (C.c_int, [vp, C.c_int, C.c_int64, vp, vp, vp, vp, vp, vp, C.c_ssize_t]),
    "b200_me_esa_host": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, vp, vp]),
}

_lib = None


def lib():
    """Load libb200dsp.so (once).  Raises B200Error when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise B200Error(f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(nvcc, sm_90a).  There is no CPU fallback.")
        L = C.CDLL(SO_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(L, name)            # AttributeError here = header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(ret, what):
    if ret is None or (isinstance(ret, int) and ret < 0):
        msg = lib().b200_last_error()
        raise B200Error(f"{what} failed ({ret}): {msg.decode() if msg else ''}")
    return ret
