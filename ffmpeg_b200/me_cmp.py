"""Host-side mirror of libavcodec's me_cmp interface (MECmpContext as filled by ff_me_cmp_init, libavcodec/me_cmp.c:961-1027)
and of the exhaustive search libavfilter drives it with (libavfilter/motion_estimation.c:78-97)."""
import ctypes as C
from ._lib import lib, check, vp, MECmpContext

SAD, SSE, PIX_ABS, HADAMARD8, VSAD, VSSE, NSSE, MEDIAN_SAD, DCT_SAD, DCT_MAX, DCT264_SAD = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10
FF_DCT_AUTO, FF_DCT_FASTINT, FF_DCT_INT, FF_DCT_FAAN = 0, 1, 2, 6                  # AVCodecContext.dct_algo (libavcodec/avcodec.h:1531-1537)
AV_CODEC_FLAG_BITEXACT = 1 << 23


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


def ff_me_cmp_init(codec_flags=AV_CODEC_FLAG_BITEXACT):
    c = MECmpContext()
    check(lib().b200_me_cmp_init(C.byref(c), codec_flags), "ff_me_cmp_init")
    return c


def me_cmp_set_dct_algo(dct_algo):
    """the forward DCT behind dct_sad / dct_max (the reference reads it from the encoder context: s->fdsp.fdct, me_cmp.c:614-622)"""
    return check(lib().b200_me_cmp_set_dct_algo(dct_algo), "me_cmp_set_dct_algo")


def me_cmp_set_nsse_weight(weight):
    """nsse's noise weight (the reference reads avctx->nsse_weight, 8 for a NULL context); process-wide, default 8"""
    lib().b200_me_cmp_set_nsse_weight(weight)


def me_cmp_batch_device(device, fn, idx, frame1, frame2, stride, h, off1, off2, n, out):
    return check(lib().b200_me_cmp_batch_device(device.handle, fn, idx, vp(_dptr(frame1)), vp(_dptr(frame2)), stride, h,
                                                vp(_dptr(off1)), vp(_dptr(off2)), n, vp(_dptr(out))), "me_cmp_batch_device")


def sum_abs_dctelem_batch_device(device, blocks, n, out):
    return check(lib().b200_sum_abs_dctelem_batch_device(device.handle, vp(_dptr(blocks)), n, vp(_dptr(out))), "sum_abs_dctelem_batch_device")


def me_esa_device(device, cur, ref, linesize, width, height, frame_stride, nframes, mb_size, search_param, out_mv, out_cost):
    return check(lib().b200_me_esa_device(device.handle, vp(_dptr(cur)), vp(_dptr(ref)), linesize, width, height, frame_stride,
                                          nframes, mb_size, search_param, vp(_dptr(out_mv)), vp(_dptr(out_cost))), "me_esa_device")


def me_esa_host(device, cur, ref, linesize, width, height, frame_stride, nframes, mb_size, search_param, out_mv, out_cost):
    """HOST buffers (numpy arrays / pinned torch tensors / raw addresses)."""
    h = lambda x: int(x.ctypes.data) if hasattr(x, "ctypes") else _dptr(x)
    return check(lib().b200_me_esa_host(device.handle, vp(h(cur)), vp(h(ref)), linesize, width, height, frame_stride,
                                        nframes, mb_size, search_param, vp(h(out_mv)), vp(h(out_cost))), "me_esa_host")


PIXELUTILS_SAD_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t)


def av_pixelutils_get_sad_fn(w_bits, h_bits, aligned=0, log_ctx=None):
    """av_pixelutils_get_sad_fn (libavutil/pixelutils.h:31-52): a function on HOST pointers, or None like the reference's NULL"""
    p = lib().b200_pixelutils_get_sad_fn(w_bits, h_bits, aligned, log_ctx)
    return PIXELUTILS_SAD_FN(p) if p else None


def pixelutils_sad_batch_device(device, w_bits, frame1, stride1, frame2, stride2, off1, off2, n, out):
    return check(lib().b200_pixelutils_sad_batch_device(device.handle, w_bits, vp(_dptr(frame1)), stride1, vp(_dptr(frame2)), stride2,
                                                        vp(_dptr(off1)), vp(_dptr(off2)), n, vp(_dptr(out))), "pixelutils_sad_batch_device")
