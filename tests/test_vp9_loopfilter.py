"""CPU tier for the VP9 loop filter (VP9DSPContext's loop-filter members and b200_vp9_loopfilter_frame_device, ffmpeg_b200/csrc/vp9lf.cu):
the checker (oracle/vp9lf_oracle.c) against the compiled reference (oracle/_ref/libffref_vp9lf.so) member by member, on whole frames at
every depth and chroma format and in wavefront orders; the fixture hashes; the fixture frames telling the superblock orders apart; the
layouts; and vp9lf.cu itself, host code included, on the stand-in CUDA runtime of tests/cuda_emu (fixture frames with sentinels, mask
bits outside the picture, every member at every depth, the init's table, refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vp9lflib as vl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38
DECODER_NAMES = [n for n in vl.FIXTURE_NAMES if n.endswith("decoder")]


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", vl.DEPTHS)
def test_checker_members_match_reference(depth):
    """all 16 members, six calls each: E / I / H over the byte range, mix2 with different halves, the 32 x 32 block around the edge"""
    ours = vl.run_members(cl.oracle(), "orc_vp9_lf_member", 30 + depth, depth)
    with vl.RefCheck() as rc:
        assert rc.same(ours, lambda: vl.run_members(vl.ref(), "ffref_vp9_lf_member", 30 + depth, depth))


@pytest.mark.parametrize("name", vl.FIXTURE_NAMES)
def test_checker_frames_match_reference(name):
    """whole frames (odd cols / rows, sizes not multiples of 64), decoder-shaped and arbitrary masks, every depth and chroma format"""
    f = vl.frame_case(name)
    ours = vl.orc_frame(f)
    assert not same(ours, f.planes)
    with vl.RefCheck() as rc:
        assert rc.same(ours, lambda: vl.ref_frame(f))


@pytest.mark.parametrize("name", ["8-420-decoder", "10-422-decoder", "12-440-arbitrary", "8-444-decoder"])
def test_checker_wavefront_orders_match_reference(name):
    """the c + r and c + 2r wavefronts (lower rows first within a step) of the checker against the reference driver's"""
    f = vl.frame_case(name)
    for k in (1, 2):
        ours = vl.orc_frame(f, k)
        with vl.RefCheck() as rc:
            assert rc.same(ours, lambda: vl.ref_frame(f, k))


def test_fixture_frames_tell_the_orders_apart():
    """the raster result equals the slope-2 wavefront, and every decoder-shaped fixture frame differs from the slope-1 wavefront and
    from the frame-wide order (all column edges, then all row edges): a frame entry that waited too little would fail its hash"""
    for name in vl.FIXTURE_NAMES:
        f = vl.frame_case(name)
        raster = vl.orc_frame(f)
        assert same(raster, vl.orc_frame(f, 2)), name
        if name in DECODER_NAMES:
            assert not same(raster, vl.orc_frame(f, 1)), name
            assert not same(raster, vl.orc_frame(f, -1)), name


def test_checker_reproduces_fixture():
    hs = vl.fixture_hashes()
    assert sorted(hs) == sorted(vl.FIXTURE_NAMES)
    for name in vl.FIXTURE_NAMES:
        assert vl.digest(vl.orc_frame(vl.frame_case(name))) == hs[name], name


def test_decoder_records_stay_in_the_picture():
    """mask_edges never sets bits of 8x8 columns >= cols or rows >= rows, its chroma 16-wide edges keep their 16 samples inside the chroma
    area and inside the superblock (never at bit 7 / row 7 of a subsampled direction), which the entry's contract relies on; the records
    reach every width and both directions"""
    seen = np.zeros((2, 2, 4), bool)
    for fmt, (ss_h, ss_v) in vl.FORMATS.items():
        for seed, (w, h) in enumerate([(328, 203), (200, 72), (72, 136), (520, 264)]):
            f = vl.Frame(seed, 8, fmt, w, h)
            arb = vl.arbitrary_records(np.random.default_rng(seed), ss_h, ss_v, f.cols, f.rows, f.lstride)
            for rec in (f.lflvl, arb):
                m = rec["mask"]
                for r in range(f.sbr):
                    for c in range(rec.shape[1]):
                        for y in range(8):
                            for k in range(8):
                                bit = (m[r, c, :, :, y, :] >> k) & 1
                                if c >= f.sbc or 8 * c + k >= f.cols or 8 * r + y >= f.rows:
                                    assert not bit.any(), (fmt, r, c, y, k)
                                elif ss_h | ss_v:
                                    x16, y16 = c * (64 >> ss_h) + k * (8 >> ss_h), r * (64 >> ss_v) + y * (8 >> ss_v)
                                    if bit[1, 0, 0]:
                                        assert x16 + 8 <= vl.area(ss_h, f.cols) and x16 != 4
                                    if bit[1, 1, 0]:
                                        assert y16 + 8 <= vl.area(ss_v, f.rows) and y16 != 4
                                    assert not (ss_h and k == 7 and bit[1, 0, 0]) and not (ss_v and y == 7 and bit[1, 1, 0])
            seen |= (f.lflvl["mask"] != 0).any(axis=(0, 1, 4))
    assert seen.all(), seen


def test_layout():
    """B200Vp9Filter / LF_DTYPE / the ctypes mirror agree (the reference build asserts the offsets against VP9Filter at compile time);
    the loop-filter members sit where VP9DSPContext has them; the reference's 16 functions are distinct"""
    from ffmpeg_b200._lib import Vp9Filter, VP9DSPContext
    from ffmpeg_b200 import vp9dsp
    assert C.sizeof(Vp9Filter) == vp9dsp.LF_DTYPE.itemsize == 192
    assert Vp9Filter.level.offset == vp9dsp.LF_DTYPE.fields["level"][1] == 0
    assert Vp9Filter.mask.offset == vp9dsp.LF_DTYPE.fields["mask"][1] == 64
    assert VP9DSPContext.loop_filter_8.offset == 80 * 8 and VP9DSPContext.loop_filter_16.offset == 86 * 8
    assert VP9DSPContext.loop_filter_mix2.offset == 88 * 8 and VP9DSPContext.mc.offset == 96 * 8
    if vl.have_ref():
        for depth in vl.DEPTHS:
            assert vl.ref().ffref_vp9_lf_distinct(depth) == 1


# ---------------------------------------------------------------- vp9lf.cu on the stand-in runtime
PROGRESS_EMU = """// ---- inter-CTA progress (stand-in: blocks run one after the other in ticket order)
static inline int ld_acquire(const int *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline void st_release(int *p, int v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline unsigned long long globaltimer() { return 0; }
static inline void __nanosleep(unsigned) {}
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
template <typename T> static inline T __ldcg(const T *p) { return *p; }
"""


def emu_source(text_fn=None):
    src = open(os.path.join(ROOT, "ffmpeg_b200", "csrc", "vp9lf.cu")).read()
    if text_fn:
        src = text_fn(src)
    a, b = src.index("// ---- inter-CTA progress\n"), src.index("// ---- end of inter-CTA progress")
    return src[:a] + PROGRESS_EMU + src[b:]


def build_emu(name, text_fn=None):
    """lib<name>.so: vp9lf.cu (after text_fn, if given) with its host code and vp9mc.cu (b200_vp9_dsp_init), compiled with g++ against
    tests/cuda_emu/fake/cuda_runtime.h.  The frame kernel's progress helpers (PTX) become host atomics, its static shared arrays statics
    (blocks run one at a time), and it runs an OS thread per CUDA thread of a block; blocks run in ticket order, so every wait is
    already satisfied."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vp9lf.cu", "vp9mc.cu", "tx_pfa.cu"):              # tx_pfa.cu: fake_device.cpp links it
        src = emu_source(text_fn) if f == "vp9lf.cu" else open(os.path.join(cs, f)).read()
        t = rewrite_launches(src)
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vp9lf.cu":
            assert t.count("emu_cfg_launch(0, [&] { vp9_lf_kernel<") == 2 and "asm" not in t
            t = t.replace("emu_cfg_launch(0, [&] { vp9_lf_kernel<", "emu_cfg_launch(2, [&] { vp9_lf_kernel<")
            t = t.replace("__shared__", "static")
        if f == "vp9mc.cu":
            t = t.replace("extern __shared__ int16_t vp9_smem[];", "int16_t *vp9_smem = (int16_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { vp9_mc_kernel<", "emu_cfg_launch(2, [&] { vp9_mc_kernel<")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, name + "_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "lib" + name + ".so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_vp9_dsp_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp9_dsp_init_loopfilter.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp9_loopfilter_frame_device.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_int64,
                                                                                  C.c_void_p, C.c_void_p]
    L.b200_vp9_loopfilter_timeouts.argtypes = [C.c_void_p, C.c_void_p]
    L.emu_launch_count.restype = C.c_uint64
    return L


@pytest.fixture(scope="module")
def emulf():
    return build_emu("emuvp9lf")


def emu_frame(L, f, lflvl=None, rec_offset=0):
    """the frame entry on copies of the planes; the records start rec_offset bytes into their buffer"""
    out = [p.copy() for p in f.planes]
    arr = (C.c_void_p * 3)(*f.ptrs(out))
    raw = np.ascontiguousarray(f.lflvl if lflvl is None else lflvl).view(np.uint8).ravel()
    buf = np.zeros(raw.size + 64, np.uint8)
    start = -buf.ctypes.data % 16 + rec_offset
    buf[start:start + raw.size] = raw
    ls_y, ls_uv = f.strides()
    assert L.b200_vp9_loopfilter_frame_device(None, f.depth, f.ss_h, f.ss_v, f.width, f.height, arr, ls_y, ls_uv, buf.ctypes.data + start,
                                              f.lstride, f.lim.ctypes.data, f.mblim.ctypes.data) == 0
    return out


def emu_timeouts(L):
    n = C.c_int64(-1)
    assert L.b200_vp9_loopfilter_timeouts(None, C.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("name", vl.FIXTURE_NAMES)
def test_emu_frame_vs_checker_and_fixture(emulf, name):
    """the fixture frame through the library's entry: equal to the checker over the whole arrays (the sentinels around every plane
    unchanged) and to the reference's hash"""
    f = vl.frame_case(name)
    got = emu_frame(emulf, f)
    assert same(got, vl.orc_frame(f))
    assert vl.digest(got) == vl.fixture_hashes()[name]
    assert emu_timeouts(emulf) == 0


@pytest.mark.parametrize("offset", (1, 2, 3))
def test_emu_records_at_any_byte_offset(emulf, offset):
    """B200Vp9Filter has byte alignment: records starting 1, 2 or 3 bytes past a word give the same frame"""
    f = vl.frame_case("10-420-arbitrary")
    assert same(emu_frame(emulf, f, rec_offset=offset), vl.orc_frame(f))


@pytest.mark.parametrize("fmt", list(vl.FORMATS))
def test_emu_ignores_bits_outside_the_picture(emulf, fmt):
    """records whose masks have bits at 8x8 columns >= cols and rows >= rows (and a longer lflvl_stride): the same picture as with
    those bits cleared, nothing outside the area written"""
    f = vl.Frame(77, 10, fmt, 136, 88, kind="arbitrary", pad=24)
    rng = np.random.default_rng(5)
    noisy = f.lflvl.copy()
    for r in range(f.sbr):
        for c in range(f.lstride):
            for y in range(8):
                for k in range(8):
                    if c >= f.sbc or 8 * c + k >= f.cols or 8 * r + y >= f.rows:
                        noisy["mask"][r, c, :, :, y, :] |= (rng.integers(0, 2, (2, 2, 4)) << k).astype(np.uint8)
    assert (noisy["mask"] != f.lflvl["mask"]).any()
    got = emu_frame(emulf, f, noisy)
    assert same(got, emu_frame(emulf, f)) and same(got, vl.orc_frame(f))


@pytest.mark.parametrize("depth", vl.DEPTHS)
def test_emu_every_member(emulf, depth):
    """every member through host pointers against the checker: the 32 x 32 block around the edge (what the member may not write
    included)"""
    from ffmpeg_b200._lib import VP9DSPContext
    ctx = VP9DSPContext()
    assert emulf.b200_vp9_dsp_init_loopfilter(C.byref(ctx), depth) == 0
    check_members(ctx, depth, 90 + depth)


def member_ptr(ctx, m):
    kind, idx = vl.MEMBERS[m]
    t = getattr(ctx, kind)
    for i in idx:
        t = t[i]
    return t


def check_members(ctx, depth, seed, per=6):
    from ffmpeg_b200.vp9dsp import VP9_LF_FUNC
    for call in vl.member_calls(seed, depth, per):
        m, E, I, H, blk = call
        d = blk.copy()
        VP9_LF_FUNC(member_ptr(ctx, m))(d.ctypes.data + 16 * d.strides[0] + 16 * d.itemsize, d.strides[0], E, I, H)
        assert np.array_equal(d, vl.run_member(cl.oracle(), "orc_vp9_lf_member", depth, call)), (depth, vl.MEMBERS[m], E, I, H)


def table_words(ctx):
    return np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)


def test_emu_init_sets_exactly_the_table(emulf):
    """on top of b200_vp9_dsp_init's context the init sets the 16 loop-filter words (80..95) and nothing else, 16 distinct functions per
    depth, different for each depth"""
    from ffmpeg_b200._lib import VP9DSPContext
    seen = set()
    for depth in vl.DEPTHS:
        ctx = VP9DSPContext()
        assert emulf.b200_vp9_dsp_init(C.byref(ctx), depth) == 0
        w0 = table_words(ctx).copy()
        assert emulf.b200_vp9_dsp_init_loopfilter(C.byref(ctx), depth) == 0
        w1 = table_words(ctx)
        assert list(np.nonzero(w0 != w1)[0]) == list(range(80, 96))
        assert len(set(w1[80:96])) == 16
        seen |= set(w1[80:96])
    assert len(seen) == 48


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emulf):
    from ffmpeg_b200._lib import VP9DSPContext
    for L in (prodlib, emulf):
        ctx = VP9DSPContext()
        for depth in (0, 7, 9, 11, 13, 14, 16):
            assert L.b200_vp9_dsp_init_loopfilter(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_vp9_dsp_init_loopfilter(None, 8) == EINVAL
        assert not table_words(ctx).any()


def test_frame_refusals(prodlib, emulf):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data + (-b.ctypes.data % 64)
    lut = np.zeros(64, np.uint8)
    before = emulf.emu_launch_count()
    for L in (prodlib, emulf):
        def call(depth=8, ss_h=1, ss_v=1, w=64, h=64, planes=(p, p + 8192, p + 12288), ls_y=64, ls_uv=32, rec=p + 16384, lstride=1,
                 lim=lut.ctypes.data, mblim=lut.ctypes.data):
            arr = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vp9_loopfilter_frame_device(None, depth, ss_h, ss_v, w, h, arr, ls_y, ls_uv, rec, lstride, lim, mblim)
        for depth in (0, 7, 9, 11, 13, 16):
            assert call(depth=depth) == EINVAL, depth
        assert call(ss_h=2) == EINVAL and call(ss_v=-1) == EINVAL
        assert call(w=0) == EINVAL and call(h=0) == EINVAL and call(w=-5) == EINVAL
        assert call(planes=None) == EINVAL and call(planes=(p, None, p)) == EINVAL and call(rec=None) == EINVAL
        assert call(lim=None) == EINVAL and call(mblim=None) == EINVAL
        assert call(ls_y=63) == EINVAL and call(ls_uv=31) == EINVAL and call(w=65, ls_y=64) == EINVAL
        assert call(ss_h=0, ls_uv=32) == EINVAL and call(w=57, ls_uv=31) == EINVAL       # chroma rows rounded up to 8 samples
        assert call(depth=10, ls_y=128, ls_uv=65) == EINVAL and call(depth=10, ls_y=129, ls_uv=64) == EINVAL
        assert call(depth=10, ls_y=128, ls_uv=64, planes=(p + 1, p + 8192, p + 12288)) == EINVAL
        assert call(depth=12, ls_y=128, ls_uv=64, planes=(p, p + 8192, p + 12289)) == EINVAL
        assert call(w=520, ls_y=1024, ls_uv=512, lstride=1) == EINVAL
        assert L.b200_vp9_loopfilter_timeouts(None, None) == EINVAL
    assert not b.any()
    assert emulf.emu_launch_count() == before
