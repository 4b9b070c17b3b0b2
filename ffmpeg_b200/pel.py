"""Host-side mirror of libavcodec's h264qpel / h264chroma / hpeldsp interfaces (H264QpelContext from ff_h264qpel_init,
libavcodec/h264qpel.c:50-120; H264ChromaContext from ff_h264chroma_init, libavcodec/h264chroma.c:36-65; HpelDSPContext from
ff_hpeldsp_init, libavcodec/hpeldsp.c:337-352) and the batched entry points."""
import ctypes as C
from ._lib import lib, check, vp, H264QpelContext, HpelDSPContext, H264ChromaContext, VideoDSPContext, H264WeightContext


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_h264qpel_init(bit_depth=8):
    c = H264QpelContext()
    check(lib().b200_h264qpel_init(C.byref(c), bit_depth), "ff_h264qpel_init")
    return c


def ff_hpeldsp_init(flags=0):
    c = HpelDSPContext()
    check(lib().b200_hpeldsp_init(C.byref(c), flags), "ff_hpeldsp_init")
    return c


def ff_h264chroma_init(bit_depth=8):
    c = H264ChromaContext()
    check(lib().b200_h264chroma_init(C.byref(c), bit_depth), "ff_h264chroma_init")
    return c


def ff_videodsp_init(bpc=8):
    """VideoDSPContext from ff_videodsp_init (libavcodec/videodsp.c:32-62): emulated_edge_mc + prefetch."""
    c = VideoDSPContext()
    check(lib().b200_videodsp_init(C.byref(c), bpc), "ff_videodsp_init")
    return c


def chroma_op(avg, idx):
    return (avg & 1) | (idx << 1)


def qpel_op(avg, size_idx, pos):
    return (avg & 1) | (size_idx << 1) | (pos << 3)


def hpel_op(tab, size_idx, xy):
    return tab | (size_idx << 2) | (xy << 4)


def h264qpel_batch_device(device, n, op, dst, dst_off, src, src_off, stride):
    return check(lib().b200_h264qpel_batch_device(device.handle, n, vp(_dptr(op)), vp(_dptr(dst)), vp(_dptr(dst_off)),
                                                  vp(_dptr(src)), vp(_dptr(src_off)), stride), "h264qpel_batch_device")


def h264qpel_hbd_batch_device(device, bit_depth, n, op, dst, dst_off, src, src_off, stride):
    """9 / 10 / 12 / 14 bit samples (uint16): offsets and stride in bytes"""
    return check(lib().b200_h264qpel_hbd_batch_device(device.handle, bit_depth, n, vp(_dptr(op)), vp(_dptr(dst)), vp(_dptr(dst_off)),
                                                      vp(_dptr(src)), vp(_dptr(src_off)), stride), "h264qpel_hbd_batch_device")


def h264qpel_frames_host(device, nframes, frame_bytes, op_begin, op, dst, dst_off, src, src_off, stride):
    """HOST buffers (numpy arrays / pinned torch tensors / raw addresses): one reference + destination picture and one operation
    list per frame, pipelined H2D -> kernel -> D2H."""
    h = lambda x: int(x.ctypes.data) if hasattr(x, "ctypes") else _dptr(x)
    return check(lib().b200_h264qpel_frames_host(device.handle, nframes, frame_bytes, vp(h(op_begin)), vp(h(op)), vp(h(dst)),
                                                 vp(h(dst_off)), vp(h(src)), vp(h(src_off)), stride), "h264qpel_frames_host")


def hpel_batch_device(device, n, op, h, dst, dst_off, src, src_off, stride):
    return check(lib().b200_hpel_batch_device(device.handle, n, vp(_dptr(op)), vp(_dptr(h)), vp(_dptr(dst)), vp(_dptr(dst_off)),
                                              vp(_dptr(src)), vp(_dptr(src_off)), stride), "hpel_batch_device")


def h264chroma_batch_device(device, n, op, h, xy, dst, dst_off, src, src_off, stride):
    return check(lib().b200_h264chroma_batch_device(device.handle, n, vp(_dptr(op)), vp(_dptr(h)), vp(_dptr(xy)), vp(_dptr(dst)),
                                                    vp(_dptr(dst_off)), vp(_dptr(src)), vp(_dptr(src_off)), stride),
                 "h264chroma_batch_device")


def h264chroma_hbd_batch_device(device, n, op, h, xy, dst, dst_off, src, src_off, stride):
    """16-bit samples (any depth above 8): offsets and stride in bytes"""
    return check(lib().b200_h264chroma_hbd_batch_device(device.handle, n, vp(_dptr(op)), vp(_dptr(h)), vp(_dptr(xy)), vp(_dptr(dst)),
                                                        vp(_dptr(dst_off)), vp(_dptr(src)), vp(_dptr(src_off)), stride),
                 "h264chroma_hbd_batch_device")


def emulated_edge_mc_hbd_batch_device(device, n, buf, buf_off, buf_linesize, src, origin, src_linesize, geom, w, h):
    """16-bit samples: geom in pixels, offsets and line sizes in bytes"""
    return check(lib().b200_emulated_edge_mc_hbd_batch_device(device.handle, n, vp(_dptr(buf)), vp(_dptr(buf_off)), buf_linesize,
                                                              vp(_dptr(src)), vp(_dptr(origin)), src_linesize, vp(_dptr(geom)), w, h),
                 "emulated_edge_mc_hbd_batch_device")


def emulated_edge_mc_batch_device(device, n, buf, buf_off, buf_linesize, src, origin, src_linesize, geom, w, h):
    """geom: int32 [n, 4] = block_w, block_h, src_x, src_y; origin: int64 offset of each window's picture sample (0, 0)."""
    return check(lib().b200_emulated_edge_mc_batch_device(device.handle, n, vp(_dptr(buf)), vp(_dptr(buf_off)), buf_linesize,
                                                          vp(_dptr(src)), vp(_dptr(origin)), src_linesize, vp(_dptr(geom)), w, h),
                 "emulated_edge_mc_batch_device")


def ff_h264dsp_weight_init(bit_depth=8):
    """weight_pixels_tab / biweight_pixels_tab as ff_h264dsp_init installs them (libavcodec/h264dsp.c:103-110)."""
    c = H264WeightContext()
    check(lib().b200_h264_weight_init(C.byref(c), bit_depth), "ff_h264dsp_init (weight)")
    return c


def weight_params(idx, height, log2_denom, weight, weights, offset):
    return [idx | (height << 8) | (log2_denom << 16), weight, weights, offset]


def h264_weight_batch_device(device, n, params, dst, dst_off, src, src_off, stride):
    """src None: weight in place; else biweight.  params: int32 [n, 4] built with weight_params()."""
    return check(lib().b200_h264_weight_batch_device(device.handle, n, vp(_dptr(params)), vp(_dptr(dst)), vp(_dptr(dst_off)),
                                                     vp(_dptr(src)) if src is not None else None,
                                                     vp(_dptr(src_off)) if src_off is not None else None, stride),
                 "h264_weight_batch_device")


def h264_weight_hbd_batch_device(device, bit_depth, n, params, dst, dst_off, src, src_off, stride):
    """9 / 10 / 12 / 14 bit samples (uint16): offsets and stride in bytes"""
    return check(lib().b200_h264_weight_hbd_batch_device(device.handle, bit_depth, n, vp(_dptr(params)), vp(_dptr(dst)), vp(_dptr(dst_off)),
                                                         vp(_dptr(src)) if src is not None else None,
                                                         vp(_dptr(src_off)) if src_off is not None else None, stride),
                 "h264_weight_hbd_batch_device")


def ff_h264dsp_loop_filter_init(bit_depth=8, chroma_format_idc=1):
    """the loop-filter members of H264DSPContext (libavcodec/h264dsp.h:48-73) on HOST pointers"""
    from ._lib import H264LoopFilterContext
    c = H264LoopFilterContext()
    check(lib().b200_h264_loop_filter_init(C.byref(c), bit_depth, chroma_format_idc), "ff_h264dsp_init (loop filter)")
    return c


def h264_loop_filter_batch_device(device, nedges, kinds, pix, pix_off, stride, alpha, beta, tc0):
    """one independent set of edges; kinds / alpha / beta uint8 [n], pix_off int64 [n], tc0 int8 [n, 4] (device)"""
    return check(lib().b200_h264_loop_filter_batch_device(device.handle, nedges, vp(_dptr(kinds)), vp(_dptr(pix)), vp(_dptr(pix_off)), stride,
                                                          vp(_dptr(alpha)), vp(_dptr(beta)), vp(_dptr(tc0))), "h264_loop_filter_batch_device")


H264_CODEC_ID = 27          # AV_CODEC_ID_H264
PRED4x4, PRED8x8L, PRED8x8, PRED8x16, PRED16x16 = range(5)                                   # b200_h264_pred_batch_device tables
PRED4x4_ADD, PRED8x8L_ADD, PRED8x8L_FILTER_ADD, PRED8x8_ADD, PRED8x16_ADD, PRED16x16_ADD = range(6)   # b200_h264_pred_add_batch_device tables


def pred_kind(table, mode):
    return (table << 4) | mode


def ff_h264_pred_init(codec_id=H264_CODEC_ID, bit_depth=8, chroma_format_idc=1):
    """H264PredContext as ff_h264_pred_init installs it (libavcodec/h264pred.c:437-539) on HOST pointers"""
    from ._lib import H264PredContext
    c = H264PredContext()
    check(lib().b200_h264_pred_init(C.byref(c), codec_id, bit_depth, chroma_format_idc), "ff_h264_pred_init")
    return c


def h264_pred_batch_device(device, bit_depth, nops, kinds, flags, pix, pix_off, stride):
    """one independent set of intra predictions; kinds / flags uint8 [n], pix_off int64 [n] in bytes (device)"""
    return check(lib().b200_h264_pred_batch_device(device.handle, bit_depth, nops, vp(_dptr(kinds)), vp(_dptr(flags)), vp(_dptr(pix)),
                                                   vp(_dptr(pix_off)), stride), "h264_pred_batch_device")


def h264_pred_add_batch_device(device, bit_depth, nops, kinds, flags, pix, pix_off, stride, coef, coef_off):
    """one independent set of lossless prediction + residual adds; coef int16 (8 bit) / int32 (above), coef_off int64 [n] in coefficients"""
    return check(lib().b200_h264_pred_add_batch_device(device.handle, bit_depth, nops, vp(_dptr(kinds)), vp(_dptr(flags)), vp(_dptr(pix)),
                                                       vp(_dptr(pix_off)), stride, vp(_dptr(coef)), vp(_dptr(coef_off))),
                 "h264_pred_add_batch_device")
