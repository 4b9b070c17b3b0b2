"""Host-side mirror of the libswscale interface for the accelerated path (yuv420p / nv12 / nv21 -> rgb24 / bgr24 / rgba / bgra / argb /
abgr / yuv420p, and packed 8-bit RGB -> yuv420p: pass the packed picture as plane 0).

Names and argument meaning follow libswscale/swscale.h: sws_getContext (:utils.c:1919), sws_setColorspaceDetails
(utils.c:849), sws_scale (swscale.c:1626), sws_freeContext.  Arrays are numpy (host) for sws_scale / scale_batch_host
and torch CUDA tensors or raw device pointers for scale_batch_device.  Everything goes through the C ABI.
"""
import ctypes as C
import numpy as np
from ._lib import lib, check, vp, i16p, i32p, i64p, B200Error, SwsFilter, SwsVector

AV_PIX_FMT_YUV420P, AV_PIX_FMT_RGB24, AV_PIX_FMT_BGR24 = 0, 2, 3                       # libavutil/pixfmt.h
AV_PIX_FMT_ARGB, AV_PIX_FMT_RGBA, AV_PIX_FMT_ABGR, AV_PIX_FMT_BGRA = 25, 26, 27, 28
AV_PIX_FMT_NV12, AV_PIX_FMT_NV21 = 23, 24                                                # source only: src[1] = interleaved chroma
SWS_FAST_BILINEAR, SWS_BILINEAR, SWS_BICUBIC, SWS_POINT, SWS_AREA, SWS_BICUBLIN = 1, 2, 4, 0x10, 0x20, 0x40
SWS_FULL_CHR_H_INT, SWS_FULL_CHR_H_INP, SWS_ACCURATE_RND, SWS_BITEXACT = 0x2000, 0x4000, 0x40000, 0x80000
# libswscale/yuv2rgb.c:47-59 (sws_getCoefficients)
SWS_CS_ITU709, SWS_CS_FCC, SWS_CS_ITU601, SWS_CS_SMPTE240M, SWS_CS_DEFAULT, SWS_CS_BT2020 = 1, 4, 5, 7, 5, 9
_BT601 = (104597, 132201, 25675, 53279)
_BT2020 = (110013, 140363, 12277, 42626)
# the reference's 11-row table (yuv2rgb.c:47-59): rows 0, 2, 3, 5, 6 are BT.601, row 8 (YCgCo) has no matrix, rows 9 and 10 are BT.2020
_COEFFS = (_BT601, (117489, 138438, 13975, 34925), _BT601, _BT601, (104448, 132798, 24759, 53109), _BT601, _BT601,
           (117579, 136230, 16907, 35559), None, _BT2020, _BT2020)


def sws_getCoefficients(colorspace):
    """yuv2rgb.c:61-66: out-of-range values and 8 (YCgCo) select SWS_CS_DEFAULT."""
    if colorspace > 10 or colorspace < 0 or colorspace == 8:
        colorspace = SWS_CS_DEFAULT
    return _COEFFS[colorspace]


def _dptr(x):
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


class SwsContext:
    def __init__(self, device, srcW, srcH, srcFormat, dstW, dstH, dstFormat, flags, src_range=0, dst_range=0, param=None, src_filter=None, dst_filter=None):
        """src_range / dst_range: SwsContext.src_range / .dst_range as set before sws_init_context (0 limited, 1 full);
        param: sws_getContext's scaler parameters (two doubles, 123456 = SWS_PARAM_DEFAULT) or None"""
        self.device = device
        self.srcW, self.srcH, self.dstW, self.dstH, self.flags = srcW, srcH, dstW, dstH, flags
        self.srcFormat, self.dstFormat = srcFormat, dstFormat
        self.dst_nv = dstFormat in (AV_PIX_FMT_NV12, AV_PIX_FMT_NV21)          # destination: luma plane + interleaved chroma plane
        self.planar = dstFormat == AV_PIX_FMT_YUV420P or self.dst_nv
        self.bpp = 1 if self.planar else 3 if dstFormat in (AV_PIX_FMT_RGB24, AV_PIX_FMT_BGR24) else 4
        pp = (C.c_double * 2)(*param) if param is not None else None
        if src_filter is not None or dst_filter is not None:
            # sws_getContext's srcFilter / dstFilter: four coefficient sequences (lumH, lumV, chrH, chrV; None = no vector) each
            keep = []

            def mk(vs):
                if vs is None:
                    return None
                f = SwsFilter()
                for name, v in zip(("lumH", "lumV", "chrH", "chrV"), vs):
                    if v is not None and len(v):
                        arr = (C.c_double * len(v))(*v)
                        vec = SwsVector(C.cast(arr, C.POINTER(C.c_double)), len(v))
                        keep.extend([arr, vec])
                        setattr(f, name, C.pointer(vec))
                keep.append(f)
                return C.byref(f)
            h = lib().b200_sws_getContext_filters(device.handle, srcW, srcH, srcFormat, src_range, dstW, dstH, dstFormat, dst_range, flags,
                                                  mk(src_filter), mk(dst_filter), pp)
        else:
            h = lib().b200_sws_getContext_params(device.handle, srcW, srcH, srcFormat, src_range, dstW, dstH, dstFormat, dst_range, flags, pp)
        if not h:
            raise B200Error("sws_getContext failed: " + lib().b200_last_error().decode())
        self._h = vp(h)

    def setColorspaceDetails(self, inv_table, srcRange, table, dstRange, brightness, contrast, saturation):
        it = (C.c_int32 * 4)(*inv_table)
        tb = (C.c_int32 * 4)(*table)
        return check(lib().b200_sws_setColorspaceDetails(self._h, it, srcRange, tb, dstRange, brightness, contrast, saturation),
                     "sws_setColorspaceDetails")

    def info(self):
        o = (C.c_int32 * 16)()
        check(lib().b200_sws_info(self._h, o), "b200_sws_info")
        return list(o)

    def last_path(self):
        """kernels used by the launches since the previous call: 1 two passes, 2 fused, 4 fused with the tensor-core horizontal pass (scaled
        path); 8 the same-size line-pair kernel"""
        return lib().b200_sws_last_path(self._h)

    def get_filter(self, which):
        info = self.info()
        size = info[which]
        n = [self.dstW, info[6], self.dstH, info[7]][which]
        if size == 0:
            return None, None, 0
        f = np.zeros(n * size, np.int16)
        p = np.zeros(n, np.int32)
        check(lib().b200_sws_get_filter(self._h, which, f.ctypes.data_as(i16p), p.ctypes.data_as(i32p), n), "get_filter")
        return f.reshape(n, size), p, size

    def scale(self, src, srcStride, srcSliceY, srcSliceH, dst, dstStride):
        """sws_scale(): src = [y,u,v] numpy uint8 arrays (or ints = host addresses), dst = [rgb]. Returns lines."""
        sp = (vp * 4)(*[a.ctypes.data if hasattr(a, "ctypes") else int(a) for a in src] + [0] * (4 - len(src)))
        ss = (C.c_int32 * 4)(*list(srcStride) + [0] * (4 - len(srcStride)))
        dp = (vp * 4)(*[a.ctypes.data if hasattr(a, "ctypes") else int(a) for a in dst] + [0] * (4 - len(dst)))
        dsr = (C.c_int32 * 4)(*list(dstStride) + [0] * (4 - len(dstStride)))
        return check(lib().b200_sws_scale(self._h, sp, ss, srcSliceY, srcSliceH, dp, dsr), "sws_scale")

    def convert(self, y, u, v, dst_pad=0):
        """Convenience: whole frame from 2-D uint8 arrays, returns (dstH, dstW*bpp+pad) array."""
        ds = self.dstW * self.bpp + dst_pad
        out = np.full((self.dstH, ds), 0xA5, np.uint8)
        n = self.scale([y, u, v], [y.strides[0], u.strides[0], v.strides[0]], 0, self.srcH, [out], [ds])   # nv12: pass the UV plane as u (v unused)
        assert n == self.dstH
        return out

    def convert_planar(self, y, u, v, dst_pad=0):
        """yuv420p destination: whole frame, returns (Y, U, V) arrays; nv12 / nv21 destination: (Y, UV)."""
        cw, ch = (self.dstW + 1) // 2, (self.dstH + 1) // 2
        dy = np.full((self.dstH, self.dstW + dst_pad), 0xA5, np.uint8)
        du = np.full((ch, (2 * cw if self.dst_nv else cw) + dst_pad), 0xA5, np.uint8)
        dv = np.full((ch, cw + dst_pad), 0xA5, np.uint8)
        dst = [dy, du] if self.dst_nv else [dy, du, dv]
        n = self.scale([y, u, v], [y.strides[0], u.strides[0], v.strides[0]], 0, self.srcH, dst, [a.strides[0] for a in dst])
        assert n == self.dstH
        return tuple(dst)

    def scale_batch_device_planar(self, src, srcStride, srcFrameStride, dst, dstStride, dstFrameStride, nframes):
        src, srcStride, srcFrameStride = (list(src) + [0] * 3)[:3], (list(srcStride) + [0] * 3)[:3], (list(srcFrameStride) + [0] * 3)[:3]
        sp = (vp * 3)(*[_dptr(a) for a in src])
        ss = (C.c_int32 * 3)(*srcStride)
        fs = (C.c_int64 * 3)(*srcFrameStride)
        dst, dstStride, dstFrameStride = (list(dst) + [0] * 3)[:3], (list(dstStride) + [0] * 3)[:3], (list(dstFrameStride) + [0] * 3)[:3]
        dp = (vp * 3)(*[_dptr(a) for a in dst])
        ds = (C.c_int32 * 3)(*dstStride)
        df = (C.c_int64 * 3)(*dstFrameStride)
        return check(lib().b200_sws_scale_batch_device_planar(self._h, sp, ss, fs, dp, ds, df, nframes), "sws_scale_batch_device_planar")

    def _batch(self, fn, src, srcStride, srcFrameStride, dst, dstStride, dstFrameStride, nframes, what):
        src, srcStride, srcFrameStride = (list(src) + [0] * 3)[:3], (list(srcStride) + [0] * 3)[:3], (list(srcFrameStride) + [0] * 3)[:3]
        sp = (vp * 3)(*[_dptr(a) for a in src])
        ss = (C.c_int32 * 3)(*srcStride)
        fs = (C.c_int64 * 3)(*srcFrameStride)
        return check(fn(self._h, sp, ss, fs, vp(_dptr(dst)), dstStride, dstFrameStride, nframes), what)

    def scale_batch_device(self, src, srcStride, srcFrameStride, dst, dstStride, dstFrameStride, nframes):
        return self._batch(lib().b200_sws_scale_batch_device, src, srcStride, srcFrameStride, dst, dstStride,
                           dstFrameStride, nframes, "sws_scale_batch_device")

    def scale_batch_host(self, src, srcStride, srcFrameStride, dst, dstStride, dstFrameStride, nframes):
        return self._batch(lib().b200_sws_scale_batch_host, src, srcStride, srcFrameStride, dst, dstStride,
                           dstFrameStride, nframes, "sws_scale_batch_host")

    def free(self):
        if self._h:
            lib().b200_sws_freeContext(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def sws_getContext(device, srcW, srcH, srcFormat, dstW, dstH, dstFormat, flags, src_range=0, dst_range=0, param=None, src_filter=None, dst_filter=None):
    return SwsContext(device, srcW, srcH, srcFormat, dstW, dstH, dstFormat, flags, src_range, dst_range, param, src_filter, dst_filter)
