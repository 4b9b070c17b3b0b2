"""GPU tier for the VP9 loop filter (ffmpeg_b200/csrc/vp9lf.cu) on the H100: b200_vp9_loopfilter_frame_device against the reference's
fixture hashes and the checker at every depth and chroma format, 3840x2160 and 1920x1080 4:2:0 frames (enough superblock rows for the
wavefront to run concurrently), a frame whose luma plane spans more than 2^31 bytes, every drop-in member through host pointers, and the
refusals.  Only committed fixtures and the checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl  # noqa: F401
import vp9lflib as vl

pytestmark = pytest.mark.gpu
EINVAL, ENOSYS = -22, -38


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def _t(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def on_device(dev, f, rec_offset=0):
    """one frame entry call on device copies of the full arrays (sentinels included), the records rec_offset bytes into their
    (256-byte aligned) buffer; returns the three arrays"""
    import torch
    from ffmpeg_b200 import vp9dsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        ts = [_t(p) for p in f.planes]
        ptrs = [t.data_ptr() + vl.MARGIN * p.strides[0] + vl.MARGIN * p.itemsize for t, p in zip(ts, f.planes)]
        raw = np.ascontiguousarray(f.lflvl).view(np.uint8).ravel()
        rec = _t(np.concatenate([np.zeros(rec_offset, np.uint8), raw]))[rec_offset:]
        ls_y, ls_uv = f.strides()
        vp9dsp.vp9_loopfilter_frame_device(dev, f.depth, f.ss_h, f.ss_v, f.width, f.height, ptrs, ls_y, ls_uv, rec, f.lstride, f.lim, f.mblim)
        dev.sync()
        return [t.cpu().numpy().view(p.dtype) for t, p in zip(ts, f.planes)]


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", vl.FIXTURE_NAMES)
def test_frame_vs_fixture(dev, name):
    """the fixture frame: the reference's three planes bit for bit (sentinels around every plane unchanged), and the checker's"""
    f = vl.frame_case(name)
    got = on_device(dev, f)
    assert vl.digest(got) == vl.fixture_hashes()[name]
    assert same(got, vl.orc_frame(f))


@pytest.mark.parametrize("depth,size", [(8, (3840, 2160)), (10, (3840, 2160)), (12, (3840, 2160)), (8, (1920, 1080)), (10, (1920, 1080))],
                         ids=("8-2160p", "10-2160p", "12-2160p", "8-1080p", "10-1080p"))
def test_large_frames(dev, depth, size):
    """4:2:0 frames with decoder-shaped records: 34 / 17 superblock rows per plane run as concurrent CTAs that wait on one another"""
    f = vl.Frame(500 + depth + size[1], depth, "420", *size)
    assert same(on_device(dev, f), vl.orc_frame(f))


def test_wavefront_repeats(dev):
    """the same 2160p frame eight times: every run equal to the checker (the CTAs' interleaving differs from run to run), and no wait
    of the whole module's frames ran out"""
    from ffmpeg_b200 import vp9dsp
    f = vl.Frame(61, 8, "420", 3840, 2160, kind="arbitrary")
    want = vl.orc_frame(f)
    for _ in range(8):
        assert same(on_device(dev, f), want)
    assert vp9dsp.vp9_loopfilter_timeouts(dev) == 0


@pytest.mark.parametrize("offset", (1, 2, 3))
def test_records_at_any_byte_offset(dev, offset):
    """B200Vp9Filter has byte alignment: a 1080p frame whose records start 1, 2 or 3 bytes past a word, equal to the checker"""
    f = vl.Frame(90 + offset, 10, "420", 1920, 1080, kind="arbitrary")
    assert same(on_device(dev, f, rec_offset=offset), vl.orc_frame(f))


def test_plane_beyond_2_31_bytes(dev):
    """a 10-bit 4:2:0 frame whose luma plane spans 2^31 + 2^27 bytes (line size 2 MiB): the samples near the end filtered like the
    checker's, the rest of every line untouched"""
    import torch
    from ffmpeg_b200 import vp9dsp
    f = vl.Frame(19, 10, "420", 264, 1088)
    ls_y, ls_uv = 1 << 21, 1 << 20
    H = f.rows * 8
    assert H * ls_y > 2 ** 31
    want = vl.orc_frame(f)
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        bufs, ptrs = [], []
        for p, (a, ls) in enumerate(zip(f.planes, (ls_y, ls_uv, ls_uv))):
            area = a[vl.MARGIN:a.shape[0] - vl.MARGIN, vl.MARGIN:a.shape[1] - vl.MARGIN]
            b = torch.zeros(area.shape[0] * ls, dtype=torch.uint8, device="cuda")
            b.view(area.shape[0], ls)[:, :area.shape[1] * 2] = _t(area).view(torch.uint8).view(area.shape[0], -1)
            bufs.append(b)
            ptrs.append(b.data_ptr())
        rec = _t(np.ascontiguousarray(f.lflvl).view(np.uint8))
        vp9dsp.vp9_loopfilter_frame_device(dev, 10, 1, 1, f.width, f.height, ptrs, ls_y, ls_uv, rec, f.lstride, f.lim, f.mblim)
        dev.sync()
        for p, (b, ls) in enumerate(zip(bufs, (ls_y, ls_uv, ls_uv))):
            w = want[p][vl.MARGIN:want[p].shape[0] - vl.MARGIN, vl.MARGIN:want[p].shape[1] - vl.MARGIN]
            rows = b.view(w.shape[0], ls)
            got = rows[:, :w.shape[1] * 2].cpu().numpy().view(np.uint16)
            assert np.array_equal(got, w), p
            assert not rows[:, w.shape[1] * 2:].any().item(), p
        del bufs
        torch.cuda.empty_cache()


@pytest.mark.parametrize("depth", vl.DEPTHS)
def test_dropin_members(dev, depth):
    """VP9DSPContext from ff_vp9dsp_init + ff_vp9dsp_init_loopfilter through the library: every loop-filter member called with host
    pointers against the checker; the mc tables untouched"""
    from ffmpeg_b200 import vp9dsp
    from test_vp9_loopfilter import check_members
    ctx = vp9dsp.ff_vp9dsp_init(depth)
    mc = bytes(ctx.mc)
    vp9dsp.ff_vp9dsp_init_loopfilter(ctx, depth)
    assert bytes(ctx.mc) == mc
    check_members(ctx, depth, 40 + depth)


def test_refusals(dev):
    """the B200_EINVAL cases of the frame entry launch nothing and write nothing"""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import VP9DSPContext
    L = fb.lib()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    lut = (C.c_uint8 * 64)()
    before = fb.launch_count()

    def call(depth=8, ss_h=1, ss_v=1, w=64, h=64, planes=(p, p + 8192, p + 12288), ls_y=64, ls_uv=32, rec=p + 16384, lstride=1):
        arr = (C.c_void_p * 3)(*planes)
        return L.b200_vp9_loopfilter_frame_device(dev.handle, depth, ss_h, ss_v, w, h, arr, ls_y, ls_uv, rec, lstride, lut, lut)
    for depth in (0, 7, 9, 11, 16):
        assert call(depth=depth) == EINVAL, depth
    assert call(ss_h=2) == EINVAL and call(w=0) == EINVAL and call(h=-1) == EINVAL and call(rec=None) == EINVAL
    assert call(planes=(p, None, p)) == EINVAL and call(ls_y=63) == EINVAL and call(ls_uv=31) == EINVAL
    assert call(depth=10, ls_y=128, ls_uv=64, planes=(p + 1, p + 8192, p + 12288)) == EINVAL and call(depth=10, ls_y=129, ls_uv=64) == EINVAL
    assert call(w=520, ls_y=1024, ls_uv=512) == EINVAL
    dev.sync()
    assert fb.launch_count() == before and not buf.any().item()
    ctx = VP9DSPContext()
    for depth in (0, 7, 9, 11, 16):
        assert L.b200_vp9_dsp_init_loopfilter(C.byref(ctx), depth) == ENOSYS, depth
    assert L.b200_vp9_dsp_init_loopfilter(None, 8) == EINVAL


def smoke(dev):
    """smoke(): a 4:2:0 frame of 3 x 3 superblocks at 8 and 10 bit, decoder-shaped records, bit-compared with the checker"""
    for depth in (8, 10):
        f = vl.Frame(3 + depth, depth, "420", 180, 150)
        assert same(on_device(dev, f), vl.orc_frame(f)), ("vp9 loop filter mismatch", depth)
