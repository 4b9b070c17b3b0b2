"""GPU tier for the VP8 / VP7 loop filter (ffmpeg_b200/csrc/vp8lf.cu) on the H100: b200_vp8_loopfilter_frame_device against the
reference's fixture hashes and the checker, seeded 1920x1088 and 3840x2160 frames (VP8 normal, VP8 simple, VP7 normal), a whole inter
frame rebuilt on the device (motion compensation, residual, loop filter), records at odd byte offsets, every drop-in member through
host pointers, and the refusals.  Only committed fixtures and the checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
import vp8dsplib as v8
import vp8lflib as vl

pytestmark = pytest.mark.gpu
EINVAL = -22


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def lf_on_device(dev, f, rec_offset=0, planes=None):
    """one frame entry call on device copies of the full arrays (sentinels included), the records rec_offset bytes into their buffer"""
    import torch
    from ffmpeg_b200 import vp8dsp
    src = planes or f.planes
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream)):
        ts = [_t(p) for p in src]
        ptrs = [t.data_ptr() + vl.MARGIN * p.strides[0] + vl.MARGIN for t, p in zip(ts, src)]
        raw = np.ascontiguousarray(f.f).view(np.uint8).ravel()
        rec = _t(np.concatenate([np.zeros(rec_offset, np.uint8), raw]))[rec_offset:]
        ls_y, ls_uv = f.strides()
        vp8dsp.vp8_loopfilter_frame_device(dev, f.is_vp7, f.simple, f.keyframe, f.mbw, f.mbh, ptrs, ls_y, ls_uv, rec, f.fstride)
        dev.sync()
        return [t.cpu().numpy() for t in ts]


@pytest.mark.parametrize("name", vl.FIXTURE_NAMES)
def test_frame_vs_fixture(dev, name):
    """the fixture frame: the reference's three planes bit for bit (sentinels around every plane unchanged), and the checker's"""
    f = vl.frame_case(name)
    got = lf_on_device(dev, f)
    assert vl.digest(got) == vl.fixture_hashes()[name]
    assert same(got, vl.orc_frame(f))


LARGE = [("vp8", 0, 0), ("vp8simple", 0, 1), ("vp7", 1, 0)]


@pytest.mark.parametrize("size", [(120, 68), (240, 135)], ids=("1920x1088", "3840x2160"))
@pytest.mark.parametrize("codec,is_vp7,simple", LARGE, ids=[c for c, _, _ in LARGE])
def test_large_frames(dev, codec, is_vp7, simple, size):
    """enough MB rows for the wavefront to run on many SMs at once: decoder-shaped records, keyframe and inter frame"""
    mbw, mbh = size
    for kf in (0, 1):
        f = vl.Frame(2000 + 3 * is_vp7 + simple + kf + mbw, mbw, mbh, is_vp7, simple, kf, "decoder", pad=32, fpad=1)
        got = lf_on_device(dev, f)
        assert same(got, vl.orc_frame(f)), (codec, kf)
        assert not same(got, f.planes)


def _orc_lf_planes(is_vp7, simple, keyframe, mbw, mbh, planes, rec, fstride):
    L = cl.oracle()
    fn = L.orc_vp8_lf_frame
    fn.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_int64, C.c_int]
    out = [p.copy() for p in planes]
    arr = (C.c_void_p * 3)(*[p.ctypes.data for p in out])
    rec = np.ascontiguousarray(rec)
    assert fn(is_vp7, simple, keyframe, mbw, mbh, arr, out[0].strides[0], out[1].strides[0], rec.ctypes.data, fstride, 0) == 0
    return out


@pytest.mark.parametrize("is_vp7,bilinear", ((0, 0), (0, 1), (1, 0)), ids=("vp8-epel", "vp8-bilinear", "vp7-epel"))
def test_inter_frame_on_device(dev, is_vp7, bilinear):
    """a whole inter frame on the device: b200_vp8_mc_frame_device, b200_vp8_residual_frame_device and the loop filter on the same
    planes in one stream, against the checker's MC, residual and loop-filter chain"""
    import torch
    from ffmpeg_b200 import vp8dsp
    mbw, mbh = 40, 23
    refs, ops, dst = v8.mc_case(3100 + is_vp7 + 2 * bilinear, mbw, mbh, intra=0.0)
    rops, coef = v8.residual_case(3110 + is_vp7, mbw, mbh, is_vp7)
    rec = vl.decoder_records(np.random.default_rng(3120 + is_vp7), mbw, mbh, mbw, is_vp7)
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream)):
        drefs = [tuple(_t(p) for p in r) for r in refs]
        dd = [_t(p) for p in dst]
        ls_y, ls_uv = dst[0].strides[0], dst[1].strides[0]
        vp8dsp.vp8_mc_frame_device(dev, bilinear, mbw, mbh, [(y, u, v, r[0].strides[0], r[1].strides[0]) for (y, u, v), r in zip(drefs, refs)],
                                   len(ops), _t(ops.view(np.uint8)), dd, ls_y, ls_uv)
        vp8dsp.vp8_residual_frame_device(dev, is_vp7, len(rops), _t(rops.view(np.uint8)), _t(coef), dd, ls_y, ls_uv)
        vp8dsp.vp8_loopfilter_frame_device(dev, is_vp7, 0, 0, mbw, mbh, dd, ls_y, ls_uv, _t(rec.view(np.uint8).ravel()), mbw)
        dev.sync()
        got = [d.cpu().numpy() for d in dd]
    exp = v8.orc_residual_frame(is_vp7, rops, coef, v8.orc_mc_frame(bilinear, mbw, mbh, refs, ops, dst))
    exp = _orc_lf_planes(is_vp7, 0, 0, mbw, mbh, exp, rec, mbw)
    assert same(got, exp)


@pytest.mark.parametrize("offset", (1, 2, 3))
def test_records_at_odd_offsets(dev, offset):
    f = vl.frame_case("vp8-kf0-arbitrary")
    assert same(lf_on_device(dev, f, rec_offset=offset), vl.orc_frame(f))


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
def test_every_member(dev, is_vp7):
    """every member through host pointers against the checker, on the two 32 x 32 blocks around the edge"""
    from ffmpeg_b200 import vp8dsp
    from test_vp8_loopfilter import check_members
    ctx = vp8dsp.ff_vp8dsp_init(is_vp7)
    vp8dsp.ff_vp8dsp_init_loopfilter(ctx, is_vp7)
    check_members(ctx, is_vp7, 70 + is_vp7)


def test_refusals(dev):
    """every B200_EINVAL case launches nothing"""
    import ffmpeg_b200 as fb
    L = fb.lib()
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data
    before = fb.launch_count()

    def call(v7=0, simple=0, kf=0, mbw=2, mbh=2, planes=(p, p + 8192, p + 12288), ls_y=32, ls_uv=16, rec=p + 16384, fstride=2):
        arr = (C.c_void_p * 3)(*planes) if planes is not None else None
        return L.b200_vp8_loopfilter_frame_device(dev.handle, v7, simple, kf, mbw, mbh, arr, ls_y, ls_uv, rec, fstride)
    assert call(planes=(p, None, p)) == EINVAL and call(rec=None) == EINVAL and call(v7=2) == EINVAL and call(simple=-1) == EINVAL
    assert call(kf=3) == EINVAL and call(mbw=0) == EINVAL and call(mbh=0) == EINVAL and call(ls_y=31) == EINVAL
    assert call(ls_uv=15) == EINVAL and call(fstride=1) == EINVAL
    assert fb.launch_count() == before and not b.any()


def test_zz_no_wait_ran_out(dev):
    """after every frame of the module, none of the kernel's bounded waits ran out on this device"""
    from ffmpeg_b200 import vp8dsp
    assert vp8dsp.vp8_loopfilter_timeouts(dev) == 0


def smoke(dev):
    """smoke(): a small frame, VP8 and VP7, normal and simple, bit-compared with the checker"""
    for is_vp7 in (0, 1):
        for simple in (0, 1):
            f = vl.Frame(41 + 2 * is_vp7 + simple, 7, 5, is_vp7, simple, simple, "decoder", pad=8, fpad=1)
            assert same(lf_on_device(dev, f), vl.orc_frame(f)), ("vp8 loop filter mismatch", is_vp7, simple)
