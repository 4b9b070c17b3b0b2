"""Test infrastructure for the VP8 / VP7 loop filter (the loop-filter members of VP8DSPContext and b200_vp8_loopfilter_frame_device):
seeded frames with decoder-shaped records (filter_level_for_mb, vp8.c:2149-2179, restated on random segmentation, loop-filter deltas,
sharpness, modes and skip flags) or arbitrary ones, member calls built to take every branch, a classifier of those branches, and runners
of the checker (oracle/liboracle.so: orc_vp8_lf_member, orc_vp8_lf_frame) and of the compiled reference (oracle/_ref/libffref_vp8lf.so,
built by oracle/ref/vp8lf.mk: ffref_vp8_lf_member, ffref_vp8_lf_frame, ffref_vp8lf_pointers).  The reference's results are kept as digests in
tests/golden/vp8lf_ref_digests.json (cpulibs.RefCheck) for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.vp8dsp import LF_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_vp8lf"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vp8lf_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vp8lf_hashes.txt")
MARGIN = 8                  # sentinel samples around every plane's area
SENTINEL = 0x5A
MODE_I4x4, VP8_MVMODE_SPLIT = 4, 7                                     # libavcodec/vp8.h:69-75
MEMBERS = ("vp8_v_loop_filter16y", "vp8_h_loop_filter16y", "vp8_v_loop_filter8uv", "vp8_h_loop_filter8uv", "vp8_v_loop_filter16y_inner",
           "vp8_h_loop_filter16y_inner", "vp8_v_loop_filter8uv_inner", "vp8_h_loop_filter8uv_inner", "vp8_v_loop_filter_simple",
           "vp8_h_loop_filter_simple")                                 # index = orc / ffref member number, context words 6..15


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


# ---------------------------------------------------------------- records
def filter_level_for_mb(p, segment, ref_frame, mode, skip, is_vp7):
    """vp8.c:2149-2179 on the frame parameters p: (filter_level, inner_limit, inner_filter)"""
    if p["seg_enabled"]:
        level = int(p["seg_level"][segment]) + (0 if p["seg_absolute"] else p["level"])
    else:
        level = p["level"]
    if p["delta_enabled"]:
        level += int(p["delta_ref"][ref_frame]) + int(p["delta_mode"][mode])
    level = min(max(level, 0), 63)
    limit = level
    if p["sharpness"]:
        limit >>= (p["sharpness"] + 3) >> 2
        limit = min(limit, 9 - p["sharpness"])
    limit = max(limit, 1)
    return level, limit, int(bool(is_vp7 or not skip or mode == MODE_I4x4 or mode == VP8_MVMODE_SPLIT))


def frame_params(rng):
    """the frame header's loop-filter fields as the decoder parses them (6-bit magnitudes with a sign, vp8.c:305-327)"""
    return {"level": int(rng.integers(0, 64)), "sharpness": int(rng.integers(0, 8)), "seg_enabled": rng.random() < 0.5,
            "seg_absolute": rng.random() < 0.5, "seg_level": rng.integers(-63, 64, 4), "delta_enabled": rng.random() < 0.6,
            "delta_ref": rng.integers(-63, 64, 4), "delta_mode": np.concatenate([np.zeros(4, np.int64), rng.integers(-63, 64, 4)])}


def decoder_records(rng, mbw, mbh, fstride, is_vp7):
    """LF_DTYPE [mbh, fstride]: per MB a segment, a reference frame, a mode that fits it (intra 0..4 with MODE_I4x4 = 4 for the current
    frame, inter 5..7 otherwise) and a skip flag, run through filter_level_for_mb; the records past mb_width hold stale values"""
    p = frame_params(rng)
    rec = np.zeros((mbh, fstride), LF_DTYPE)
    for name in LF_DTYPE.names:
        rec[name] = rng.integers(0, 256, rec.shape)
    for y in range(mbh):
        for x in range(mbw):
            ref = int(rng.choice(4, p=[0.2, 0.5, 0.15, 0.15]))
            mode = int(rng.integers(0, 5)) if ref == 0 else int(rng.integers(5, 8))
            rec[y, x] = filter_level_for_mb(p, int(rng.integers(0, 4)), ref, mode, rng.random() < 0.4, is_vp7)
    return rec


def arbitrary_records(rng, mbw, mbh, fstride):
    """levels 0..63 and some above (left untouched), any inner_limit, inner_filter 0, 1 or 2..255"""
    rec = np.zeros((mbh, fstride), LF_DTYPE)
    lvl = rng.integers(0, 64, rec.shape)
    big = rng.random(rec.shape) < 0.06
    lvl[big] = rng.integers(64, 256, int(big.sum()))
    lvl[rng.random(rec.shape) < 0.06] = 0
    rec["filter_level"] = lvl
    rec["inner_limit"] = np.where(rng.random(rec.shape) < 0.7, rng.integers(0, 20, rec.shape), rng.integers(0, 256, rec.shape))
    rec["inner_filter"] = rng.choice(np.array([0, 1, 1, 2, 77, 255]), rec.shape)
    return rec


# ---------------------------------------------------------------- frames
def content(rng, h, w):
    """4x4 blocks of a smooth base with steps between them and per-block noise of several amplitudes, so that the limits, hev and the
    clips all go both ways"""
    by, bx = (h + 3) // 4, (w + 3) // 4
    yy, xx = np.mgrid[0:by, 0:bx]
    base = 128 + 90 * np.sin(xx / 3.0 + yy / 5.0) + rng.integers(-20, 21, (by, bx)) * (rng.random((by, bx)) < 0.6)
    base[rng.random((by, bx)) < 0.05] = 0
    base[rng.random((by, bx)) < 0.05] = 255
    amp = rng.choice([0, 0, 1, 2, 4, 8, 40], (by, bx))
    img = np.kron(base, np.ones((4, 4)))[:h, :w]
    noise = rng.integers(-(1 << 20), 1 << 20, (h, w)) % (np.kron(amp, np.ones((4, 4), np.int64))[:h, :w] + 1)
    return np.clip(img + noise - np.kron(amp, np.ones((4, 4), np.int64))[:h, :w] // 2, 0, 255).astype(np.uint8)


class Frame:
    """one frame: three planes (full arrays with MARGIN sentinel samples around the area, `pad` more columns right of it: strides wider
    than the plane), records LF_DTYPE [mb_height, f_stride] with f_stride = mb_width + fpad"""

    def __init__(self, seed, mbw, mbh, is_vp7, simple, keyframe, kind="decoder", pad=0, fpad=0):
        rng = np.random.default_rng(seed)
        self.mbw, self.mbh, self.is_vp7, self.simple, self.keyframe = mbw, mbh, is_vp7, simple, keyframe
        self.planes = []
        for s in (16, 8, 8):
            a = np.full((s * mbh + 2 * MARGIN, s * mbw + 2 * MARGIN + pad), SENTINEL, np.uint8)
            a[MARGIN:MARGIN + s * mbh, MARGIN:MARGIN + s * mbw] = content(rng, s * mbh, s * mbw)
            self.planes.append(a)
        self.fstride = mbw + fpad
        self.f = (decoder_records(rng, mbw, mbh, self.fstride, is_vp7) if kind == "decoder" else
                  arbitrary_records(rng, mbw, mbh, self.fstride))

    def ptrs(self, planes):
        return [p.ctypes.data + MARGIN * p.strides[0] + MARGIN for p in planes]

    def strides(self):
        return self.planes[0].strides[0], self.planes[1].strides[0]

    def area(self, planes):
        """the planes' areas (views)"""
        return [p[MARGIN:MARGIN + s * self.mbh, MARGIN:MARGIN + s * self.mbw] for p, s in zip(planes, (16, 8, 8))]


def _frame(L, name, f, extra, planes=None):
    fn = getattr(L, name)
    fn.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_int64] + [C.c_int] * len(extra)
    out = [p.copy() for p in (planes or f.planes)]
    arr = (C.c_void_p * 3)(*f.ptrs(out))
    rec = np.ascontiguousarray(f.f)
    ls_y, ls_uv = f.strides()
    assert fn(f.is_vp7, f.simple, f.keyframe, f.mbw, f.mbh, arr, ls_y, ls_uv, rec.ctypes.data, f.fstride, *extra) == 0
    return out


def orc_frame(f, order=0, planes=None):
    """the checker: order 0 raster (the entry's result), k >= 1 wavefront c + k r, -1 frame-wide columns then rows, -2 VP8's edge
    order"""
    return _frame(cl.oracle(), "orc_vp8_lf_frame", f, (order,), planes)


def ref_frame(f, planes=None):
    """the reference members in the decoder's raster sequence"""
    return _frame(ref(), "ffref_vp8_lf_frame", f, (), planes)


# ---------------------------------------------------------------- fixture frames
CODECS = {"vp8": (0, 0), "vp8simple": (0, 1), "vp7": (1, 0), "vp7simple": (1, 1)}     # (is_vp7, simple)
FIXTURE_NAMES = [f"{c}-kf{k}-{kind}" for c in CODECS for k in (0, 1) for kind in ("decoder", "arbitrary")]


def frame_case(name):
    """the frames behind tests/golden/vp8lf_hashes.txt: name = '<codec>-kf<keyframe>-<kind>'; 11 x 7 macroblocks, planes 24 columns
    wider than the area, records 2 wider than a row"""
    codec, kf, kind = name.split("-")
    is_vp7, simple = CODECS[codec]
    seed = 1200 + 10 * list(CODECS).index(codec) + 2 * int(kf[2:]) + (kind != "decoder")
    return Frame(seed, 11, 7, is_vp7, simple, int(kf[2:]), kind, pad=24, fpad=2)


def digest(planes):
    h = hashlib.sha256()
    for p in planes:
        h.update(np.ascontiguousarray(p).tobytes())
    return h.hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        name, h = line.split()
        out[name] = h
    return out


# ---------------------------------------------------------------- members
def member_geometry(m):
    """(dir, kind, uv) of member m: dir 1 = v (edge between rows), kind 0 MB edge, 1 inner, 2 simple"""
    return (0 if m & 1 else 1), (2 if m >= 8 else 1 if m >= 4 else 0), (m < 8 and bool(m & 2))


def member_calls(seed, is_vp7, per=12):
    """(member, E, I, H, blocks [2][32, 32] with q0 of line 0 at (16, 16); the second block is V for 8uv) for all ten members: each line
    across the edge built from one of several shapes (flat with noise, steps of every size, extremes, the pattern that gives
    a = 124 in filter_common, where VP7's f2 differs from VP8's), E / I / H mostly near the lines' own differences, some over the byte
    range"""
    rng = np.random.default_rng(seed)
    for m in range(10):
        dir, kind, uv = member_geometry(m)
        for it in range(per):
            blks = []
            for _ in range(2):
                b = rng.integers(0, 256, (32, 32)).astype(np.int64)
                for ln in range(16):
                    shape = int(rng.integers(0, 6))
                    base = int(rng.integers(0, 256))
                    if shape == 0:                                      # flat with small noise and a step
                        v = base + rng.integers(-2, 3, 8) + np.where(np.arange(8) >= 4, int(rng.integers(-30, 31)), 0)
                    elif shape == 1:                                    # extremes: 0 / 255 on either side
                        v = np.where(np.arange(8) >= 4, int(rng.choice([0, 255])), int(rng.choice([0, 255]))) + rng.integers(-3, 4, 8)
                    elif shape == 2:                                    # a = 3 (q0 - p0) + (p1 - q1) = 124
                        p0 = int(rng.integers(0, 200))
                        q0, p1 = p0 + 41, p0 + int(rng.integers(-2, 3))
                        v = np.array([p1, p1, p1, p0, q0, p1 - 1, p1 - 1, p1 - 1])
                    elif shape == 3:                                    # large swings: clip_int8 both ways
                        v = np.array([base] * 3 + [int(rng.integers(0, 256)), int(rng.integers(0, 256))] + [255 - base] * 3)
                    else:                                               # smooth ramps
                        v = base + np.arange(8) * int(rng.integers(-6, 7)) + rng.integers(-1, 2, 8)
                    v = np.clip(v, 0, 255)
                    if dir:
                        b[12:20, 16 + ln] = v
                    else:
                        b[16 + ln, 12:20] = v
                blks.append(b.astype(np.uint8))
            if it % 4 == 3:
                E, I, H = (int(v) for v in rng.integers(0, 256, 3))
            else:
                E, I, H = int(rng.integers(0, 140)), int(rng.integers(0, 40)), int(rng.integers(0, 12))
            yield m, E, I, H, np.stack(blks)


def run_member(L, name, is_vp7, call):
    m, E, I, H, blks = call
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int]
    d = blks.copy()
    assert f(is_vp7, m, d[0].ctypes.data + 16 * 32 + 16, d[1].ctypes.data + 16 * 32 + 16, 32, E, I, H) == 0
    return d


def run_members(L, name, seed, is_vp7):
    return [run_member(L, name, is_vp7, c) for c in member_calls(seed, is_vp7)]


def branches(is_vp7, call):
    """which branches the lines of a member call take, from its input alone: a set of names ('limit-false', 'limit-true', 'hev-false',
    'hev-true', 'int8-low', 'int8-high', 'u8-low', 'u8-high', 'a124')"""
    m, E, I, H, blks = call
    dir, kind, uv = member_geometry(m)
    seen = set()
    for b in blks[:2 if uv else 1]:
        for ln in range(8 if uv else 16):
            v = (b[12:20, 16 + ln] if dir else b[16 + ln, 12:20]).astype(np.int64)
            p3, p2, p1, p0, q0, q1, q2, q3 = v
            ok = (abs(p0 - q0) <= E) if is_vp7 else (2 * abs(p0 - q0) + (abs(p1 - q1) >> 1) <= E)
            if kind != 2:
                ok = ok and max(abs(p3 - p2), abs(p2 - p1), abs(p1 - p0), abs(q3 - q2), abs(q2 - q1), abs(q1 - q0)) <= I
            seen.add("limit-true" if ok else "limit-false")
            if not ok:
                continue
            hev = kind == 2 or abs(p1 - p0) > H or abs(q1 - q0) > H
            seen.add("hev-true" if hev else "hev-false")
            raw = 3 * (q0 - p0) + (np.clip(p1 - q1, -128, 127) if (hev or kind == 0) else 0)
            if raw < -128 or (hev or kind == 0) and p1 - q1 < -128:
                seen.add("int8-low")
            if raw > 127 or (hev or kind == 0) and p1 - q1 > 127:
                seen.add("int8-high")
            a = int(np.clip(raw, -128, 127))
            if hev or kind != 0:
                seen.add("a124") if a == 124 and hev else None
                f1 = min(a + 4, 127) >> 3
                outs = [p0 + f1, q0 - f1]
            else:
                w = a
                outs = [p0 + ((27 * w + 63) >> 7), q0 - ((27 * w + 63) >> 7), p2 + ((9 * w + 63) >> 7), q2 - ((9 * w + 63) >> 7)]
            if min(outs) < 0:
                seen.add("u8-low")
            if max(outs) > 255:
                seen.add("u8-high")
    return seen
