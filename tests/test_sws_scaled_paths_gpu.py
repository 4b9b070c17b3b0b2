"""GPU tier: the scaled path's three kernels — the fused tensor-core kernels (csrc/sws_mma.cuh), the fused CUDA-core kernels and the two passes
through int16 line planes — on the same cases (tests/cases.py SWS_PATH_CASES), bit for bit against the oracle.

Every case runs through the batched device entry points in three memory layouts, one call each:
  A: every plane's base, row stride and frame stride a multiple of 16, rows and frames padded: the tensor-core kernels wherever the shape allows;
  B: source planes at base + 1 with odd row and frame strides, destination as in A: the CUDA-core fused kernels where the filters have at most
     16 taps, else two passes;
  C: destination at base + 1 with odd row and frame strides: two passes.
Each call asserts the kernel the case's row names (b200_sws_last_path), that every frame equals the oracle's, that the padding between rows,
between frames and the 256 bytes past the batch still hold their sentinel, and that the source buffers are unchanged.  One more call per
layout carries 65537 frames, more than one launch's gridDim.z, with a period of 7 inputs that does not divide the 65535-frame chunks."""
import numpy as np
import pytest

import cpulibs as cl
from cases import SWS_PATH_CASES, FATE

pytestmark = pytest.mark.gpu

KINDS = ("random", "smooth", "limited", "extremes")
FMT = {"yuv420p": 0, **cl.PACKED_RGB_FORMATS}
LAYOUTS = "ABC"
SENTINEL, SRC_FILL, TAIL = 0xA5, 0x5A, 256


def plane_layout(width, h, n, misaligned):
    """(byte offset of frame 0, row stride, frame stride, buffer bytes) of n frames of h rows of `width` bytes"""
    if misaligned:
        off, rs = 1, (width + 3) | 1
        fs = rs * h + 7
    else:
        off, rs = 0, ((width + 15) & ~15) + 16
        fs = rs * h + 48
    return off, rs, fs, off + fs * (n - 1) + rs * h + TAIL


def frames_view(flat, off, rs, fs, n, h, width):
    return np.lib.stride_tricks.as_strided(flat[off:], shape=(n, h, width), strides=(fs, rs, 1))


class Planes:
    """n frames of one set of planes in flat buffers laid out by plane_layout(); widths in bytes"""

    def __init__(self, widths, heights, n, misaligned, fill):
        self.geo = [plane_layout(w, h, n, misaligned) for w, h in zip(widths, heights)]
        self.flat = [np.full(g[3], fill, np.uint8) for g in self.geo]
        self.shape = list(zip(heights, widths))
        self.n = n

    def view(self, k):
        off, rs, fs, _ = self.geo[k]
        return frames_view(self.flat[k], off, rs, fs, self.n, *self.shape[k])

    def stride(self, k):
        return self.geo[k][1]

    def fstride(self, k):
        return self.geo[k][2]


def case_frames(row, kinds=KINDS, seed0=0):
    """per input kind: the source planes as the entry points take them (y, u, v or y, uv) and as the oracle takes them (y, u, v)"""
    w, h = row["geom"][:2]
    sf = row.get("src_fmt", 0)
    out = []
    for i, kind in enumerate(kinds):
        y, u, v = cl.yuv_frame(w, h, seed0 + 70 + i, kind)
        if sf:
            uv = cl.nv_interleave(u, v, sf)
            out.append(((y, uv), (y, uv, uv)))
        else:
            out.append(((y, u, v), (y, u, v)))
    return out


def oracle_out(row, dest, planes):
    w, h, dw, dh = row["geom"]
    kw = dict(src_fmt=row.get("src_fmt", 0), param=row.get("param"))
    if row.get("src_filter"):
        kw["filters"] = (row["src_filter"], None)
    if dest == "yuv420p":
        return cl.orc_sws_planar(w, h, dw, dh, row["flags"], *planes, **kw)
    return (cl.orc_sws(w, h, dw, dh, row["flags"], *planes, fmt=FMT[dest], **kw),)


def dst_shapes(row, dest):
    dw, dh = row["geom"][2:]
    if dest == "yuv420p":
        cw, ch = (dw + 1) // 2, (dh + 1) // 2
        return [dw, cw, cw], [dh, ch, ch]
    return [dw * cl.fmt_bpp(FMT[dest])], [dh]


def run_layout(device, row, dest, layout, src_frames, exp_frames, index):
    """one batched call of len(index) frames (frame f takes src_frames[index[f]]) in `layout`; returns b200_sws_last_path and checks
    destination (exp_frames[index[f]] per frame, sentinels elsewhere) and source buffers"""
    import torch
    from ffmpeg_b200 import swscale as sw
    w, h, dw, dh = row["geom"]
    n = len(index)
    src_w = [a.shape[1] for a in src_frames[0]]
    src_h = [a.shape[0] for a in src_frames[0]]
    S = Planes(src_w, src_h, n, layout == "B", SRC_FILL)
    for k in range(len(src_w)):
        S.view(k)[:] = np.stack([f[k] for f in src_frames])[index]
    dws, dhs = dst_shapes(row, dest)
    D = Planes(dws, dhs, n, layout == "C", SENTINEL)
    E = Planes(dws, dhs, n, layout == "C", SENTINEL)
    for k in range(len(dws)):
        E.view(k)[:] = np.stack([f[k] for f in exp_frames])[index]
    ctx = sw.sws_getContext(device, w, h, row.get("src_fmt", 0), dw, dh, FMT[dest], row["flags"], param=row.get("param"),
                            src_filter=row.get("src_filter"))
    with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
        ds = [torch.from_numpy(a).cuda() for a in S.flat]
        dd = [torch.from_numpy(a).cuda() for a in D.flat]
        sp = [int(t.data_ptr()) + S.geo[k][0] for k, t in enumerate(ds)]
        dp = [int(t.data_ptr()) + D.geo[k][0] for k, t in enumerate(dd)]
        sst, sfs = [S.stride(k) for k in range(len(ds))], [S.fstride(k) for k in range(len(ds))]
        if dest == "yuv420p":
            ctx.scale_batch_device_planar(sp, sst, sfs, dp, [D.stride(k) for k in range(3)], [D.fstride(k) for k in range(3)], n)
        else:
            ctx.scale_batch_device(sp, sst, sfs, dp[0], D.stride(0), D.fstride(0), n)
        device.sync()
        got_d = [t.cpu().numpy() for t in dd]
        got_s = [t.cpu().numpy() for t in ds]
    path = ctx.last_path()
    ctx.free()
    for k in range(len(dws)):
        if not np.array_equal(got_d[k], E.flat[k]):
            bad = np.flatnonzero(got_d[k] != E.flat[k])
            off, rs, fs, _ = D.geo[k]
            f, r = divmod(int(bad[0]) - off, fs)
            raise AssertionError(f"layout {layout} plane {k}: {bad.size} bytes differ, first at frame {f} row {r // rs} byte {r % rs} "
                                 f"(row bytes {dws[k]}, frames {n}), path {path}")
    for k in range(len(src_w)):
        assert np.array_equal(got_s[k], S.flat[k]), (layout, "source plane changed", k)
    return path


def case_id(row, dest):
    w, h, dw, dh = row["geom"]
    extra = {23: "_nv12", 24: "_nv21"}.get(row.get("src_fmt", 0), "") + ("_param" if row.get("param") else "") + \
        ("_srcfilter" if row.get("src_filter") else "")
    return f"{w}x{h}-{dw}x{dh}-{row['flags']:x}{extra}-{dest}"


PARAMS = [(row, dest) for row in SWS_PATH_CASES for dest in row["paths"]]


@pytest.mark.parametrize("row,dest", PARAMS, ids=[case_id(r, d) for r, d in PARAMS])
def test_scaled_path_case(device, row, dest):
    frames = case_frames(row)
    src = [f[0] for f in frames]
    exp = [oracle_out(row, dest, f[1]) for f in frames]
    index = np.arange(len(frames))
    got = tuple(run_layout(device, row, dest, lay, src, exp, index) for lay in LAYOUTS)
    assert got == row["paths"][dest], ("kernels (A, B, C)", got, "expected", row["paths"][dest])


CHUNK_ROW = dict(geom=(64, 36, 32, 18), flags=FATE)
CHUNK_PATHS = {"rgb24": (4, 2, 1), "yuv420p": (4, 2, 1)}


@pytest.mark.parametrize("dest", sorted(CHUNK_PATHS))
def test_frames_beyond_one_launch(device, dest):
    """65537 frames in one call: the entry points split them into launches of at most 65535 (gridDim.z); frame f takes input f % 7,
    so a chunk that lost its frame offset reads or writes the wrong frame"""
    kinds = ("random", "smooth", "limited", "extremes", "random", "random", "smooth")
    frames = case_frames(CHUNK_ROW, kinds, seed0=900)
    src = [f[0] for f in frames]
    exp = [oracle_out(CHUNK_ROW, dest, f[1]) for f in frames]
    index = np.arange(65537) % 7
    got = tuple(run_layout(device, CHUNK_ROW, dest, lay, src, exp, index) for lay in LAYOUTS)
    assert got == CHUNK_PATHS[dest], got
