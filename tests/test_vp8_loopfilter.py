"""CPU tier for the VP8 / VP7 loop filter (VP8DSPContext's loop-filter members and b200_vp8_loopfilter_frame_device,
ffmpeg_b200/csrc/vp8lf.cu): the checker (oracle/vp8lf_oracle.c) against the compiled reference (oracle/_ref/libffref_vp8lf.so) member by
member with every branch taken, and on whole frames of every codec and filter type; the fixture hashes; the fixture frames telling the
macroblock orders apart; the layouts; and vp8lf.cu itself, host code included, on the stand-in CUDA runtime of tests/cuda_emu (fixture
frames with sentinels, records at every byte offset, levels above 63, chroma under the simple filter, every member, the init's table,
refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vp8lflib as vl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL = -22
DECODER_NAMES = [n for n in vl.FIXTURE_NAMES if n.endswith("decoder")]
BRANCHES = {"limit-false", "limit-true", "hev-false", "hev-true", "int8-low", "int8-high", "u8-low", "u8-high", "a124"}


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
def test_checker_members_match_reference(is_vp7):
    """all ten members, twelve calls each, on lines built so that the simple / normal limit is false and true, hev false and true,
    clip_int8 clips at both bounds, the output clips at 0 and 255, and a = 124 (where VP7's f2 differs from VP8's) all occur"""
    seen = set()
    for call in vl.member_calls(20 + is_vp7, is_vp7):
        seen |= vl.branches(is_vp7, call)
    assert seen == BRANCHES, BRANCHES - seen
    ours = vl.run_members(cl.oracle(), "orc_vp8_lf_member", 20 + is_vp7, is_vp7)
    with vl.RefCheck() as rc:
        assert rc.same(ours, lambda: vl.run_members(vl.ref(), "ffref_vp8_lf_member", 20 + is_vp7, is_vp7))


@pytest.mark.parametrize("name", vl.FIXTURE_NAMES)
def test_checker_frames_match_reference(name):
    """the fixture frames: VP8 and VP7, normal and simple, keyframe 0 and 1, decoder-shaped and arbitrary records, strides wider than
    the plane and a record stride wider than mb_width"""
    f = vl.frame_case(name)
    ours = vl.orc_frame(f)
    assert not same(ours, f.planes)
    with vl.RefCheck() as rc:
        assert rc.same(ours, lambda: vl.ref_frame(f))


SHAPES = [(1, 1), (1, 9), (9, 1), (3, 2), (24, 3)]


@pytest.mark.parametrize("mbw,mbh", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_checker_frame_shapes_match_reference(mbw, mbh):
    """1x1, 1xN and Nx1 macroblock frames and small ones, every codec and filter type, both kinds of record"""
    outs = []
    for k, (codec, (is_vp7, simple)) in enumerate(vl.CODECS.items()):
        for kind in ("decoder", "arbitrary"):
            f = vl.Frame(300 + 7 * mbw + mbh + 2 * k + (kind == "decoder"), mbw, mbh, is_vp7, simple, k & 1, kind, pad=mbw % 5, fpad=mbh % 3)
            outs.append((f, vl.orc_frame(f)))
    with vl.RefCheck() as rc:
        for f, ours in outs:
            assert rc.same(ours, lambda: vl.ref_frame(f))


def test_fixture_frames_tell_the_orders_apart():
    """the raster result equals the slope-2 wavefront, and every decoder-shaped fixture frame differs from a slope-1 wavefront and from
    the frame-wide order (all column edges, then all row edges), and each VP7 normal one from VP8's edge order: a frame entry that
    waited too little or ordered the edges wrongly fails its hash"""
    for name in vl.FIXTURE_NAMES:
        f = vl.frame_case(name)
        raster = vl.orc_frame(f)
        assert same(raster, vl.orc_frame(f, 2)), name
        if name in DECODER_NAMES:
            assert not same(raster, vl.orc_frame(f, 1)), name
            assert not same(raster, vl.orc_frame(f, -1)), name
            if f.is_vp7 and not f.simple:
                assert not same(raster, vl.orc_frame(f, -2)), name


def test_checker_reproduces_fixture():
    hs = vl.fixture_hashes()
    assert sorted(hs) == sorted(vl.FIXTURE_NAMES)
    for name in vl.FIXTURE_NAMES:
        assert vl.digest(vl.orc_frame(vl.frame_case(name))) == hs[name], name


def test_decoder_records():
    """filter_level_for_mb's records: levels 0..63, inner_limit 1..63 and at most the level (or 1), inner_filter 0 / 1 (always 1 for VP7),
    the levels spread over the range"""
    levels = set()
    for is_vp7 in (0, 1):
        for seed in range(12):
            rec = vl.decoder_records(np.random.default_rng(seed), 20, 6, 20, is_vp7)
            assert (rec["filter_level"] <= 63).all() and (rec["inner_limit"] >= 1).all()
            assert (rec["inner_limit"] <= np.maximum(rec["filter_level"], 1)).all()
            assert set(np.unique(rec["inner_filter"])) <= ({1} if is_vp7 else {0, 1})
            levels |= set(int(v) for v in rec["filter_level"].ravel())
    assert {0, 63} <= levels and len(levels) >= 32


def test_layout():
    """B200Vp8FilterStrength / LF_DTYPE / the ctypes mirror agree (the reference build asserts the offsets against VP8FilterStrength at
    compile time); the loop-filter members sit where VP8DSPContext has them"""
    from ffmpeg_b200._lib import Vp8FilterStrength, VP8DSPContext
    from ffmpeg_b200 import vp8dsp
    assert C.sizeof(Vp8FilterStrength) == vp8dsp.LF_DTYPE.itemsize == 3
    for name, _ in Vp8FilterStrength._fields_:
        assert getattr(Vp8FilterStrength, name).offset == vp8dsp.LF_DTYPE.fields[name][1], name
    for k, name in enumerate(vl.MEMBERS):
        assert getattr(VP8DSPContext, name).offset == (6 + k) * 8, name
    assert C.sizeof(VP8DSPContext) == 70 * 8 and VP8DSPContext.put_vp8_epel_pixels_tab.offset == 16 * 8
    if vl.have_ref():
        marker = C.c_char_p.in_dll(vl.ref(), "ffref_vp8lf_layout_check")
        assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200Vp8FilterStrength matches")


# ---------------------------------------------------------------- vp8lf.cu on the stand-in runtime
PROGRESS_EMU = """// ---- inter-CTA progress (stand-in: blocks run one after the other in ticket order)
static inline int ld_acquire(const int *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline void st_release(int *p, int v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline unsigned long long globaltimer() { return 0; }
static inline void __nanosleep(unsigned) {}
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
template <typename T> static inline T __ldcg(const T *p) { return *p; }
"""


def emu_source(text_fn=None):
    src = open(os.path.join(ROOT, "ffmpeg_b200", "csrc", "vp8lf.cu")).read()
    if text_fn:
        src = text_fn(src)
    a, b = src.index("// ---- inter-CTA progress\n"), src.index("// ---- end of inter-CTA progress")
    return src[:a] + PROGRESS_EMU + src[b:]


def build_emu(name, text_fn=None):
    """lib<name>.so: vp8lf.cu (after text_fn, if given) with its host code, vp8mc.cu and vp8idct.cu (b200_vp8_dsp_init), compiled with
    g++ against tests/cuda_emu/fake/cuda_runtime.h.  The frame kernel's progress helpers (PTX) become host atomics, its static shared
    arrays statics (blocks run one at a time), __syncwarp the warp's barrier, and it runs an OS thread per CUDA thread of a block; blocks
    run in ticket order, so every wait is already satisfied."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vp8lf.cu", "vp8mc.cu", "vp8idct.cu", "tx_pfa.cu"):      # tx_pfa.cu: fake_device.cpp links it
        src = emu_source(text_fn) if f == "vp8lf.cu" else open(os.path.join(cs, f)).read()
        t = rewrite_launches(src)
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vp8lf.cu":
            assert t.count("emu_cfg_launch(0, [&] { vp8_lf_kernel(") == 1 and "asm" not in t
            t = t.replace("emu_cfg_launch(0, [&] { vp8_lf_kernel(", "emu_cfg_launch(2, [&] { vp8_lf_kernel(")
            t = t.replace("__shared__", "static")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        if f == "vp8mc.cu":
            t = t.replace("extern __shared__ uint32_t vp8_smem[];", "uint32_t *vp8_smem = (uint32_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { vp8_mc_kernel(", "emu_cfg_launch(2, [&] { vp8_mc_kernel(")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, name + "_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "lib" + name + ".so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=",
                        "-I" + os.path.join(EMU, "fake"), "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs +
                       [os.path.join(EMU, "fake_device.cpp"), "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_vp8_dsp_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp8_dsp_init_loopfilter.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp8_loopfilter_frame_device.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_int64]
    L.b200_vp8_loopfilter_timeouts.argtypes = [C.c_void_p, C.c_void_p]
    L.emu_launch_count.restype = C.c_uint64
    return L


@pytest.fixture(scope="module")
def emulf():
    return build_emu("emuvp8lf")


def emu_frame(L, f, rec=None, rec_offset=0, planes=None):
    """the frame entry on copies of the planes; the records start rec_offset bytes past a 16-byte boundary of their buffer"""
    out = [p.copy() for p in (planes or f.planes)]
    arr = (C.c_void_p * 3)(*f.ptrs(out))
    raw = np.ascontiguousarray(f.f if rec is None else rec).view(np.uint8).ravel()
    buf = np.zeros(raw.size + 64, np.uint8)
    start = -buf.ctypes.data % 16 + rec_offset
    buf[start:start + raw.size] = raw
    ls_y, ls_uv = f.strides()
    assert L.b200_vp8_loopfilter_frame_device(None, f.is_vp7, f.simple, f.keyframe, f.mbw, f.mbh, arr, ls_y, ls_uv, buf.ctypes.data + start,
                                              f.fstride) == 0
    return out


def emu_timeouts(L):
    n = C.c_int64(-1)
    assert L.b200_vp8_loopfilter_timeouts(None, C.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("name", vl.FIXTURE_NAMES)
def test_emu_frame_vs_checker_and_fixture(emulf, name):
    """the fixture frame through the library's entry: equal to the checker over the whole arrays (the sentinels around every plane and
    in the padding unchanged) and to the reference's hash"""
    f = vl.frame_case(name)
    got = emu_frame(emulf, f)
    assert same(got, vl.orc_frame(f))
    assert vl.digest(got) == vl.fixture_hashes()[name]
    assert emu_timeouts(emulf) == 0


@pytest.mark.parametrize("mbw,mbh", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_emu_frame_shapes(emulf, mbw, mbh):
    for k, (codec, (is_vp7, simple)) in enumerate(vl.CODECS.items()):
        f = vl.Frame(400 + 7 * mbw + mbh + k, mbw, mbh, is_vp7, simple, k & 1, "arbitrary" if k & 2 else "decoder", pad=mbw % 5, fpad=mbh % 3)
        assert same(emu_frame(emulf, f), vl.orc_frame(f)), codec


@pytest.mark.parametrize("offset", (0, 1, 2, 3))
def test_emu_records_at_any_byte_offset(emulf, offset):
    """the records are 3 bytes at every alignment: starting 0..3 bytes past a word gives the same frame"""
    f = vl.frame_case("vp7-kf0-arbitrary")
    assert same(emu_frame(emulf, f, rec_offset=offset), vl.orc_frame(f))


def test_emu_levels_above_63_untouched(emulf):
    """MBs with filter_level > 63 are left as they are: with every level above 63 nothing changes, and an MB above 63 amid filtered ones
    gives the checker's frame (which skips them)"""
    for is_vp7, simple in vl.CODECS.values():
        f = vl.Frame(500 + 2 * is_vp7 + simple, 5, 4, is_vp7, simple, 0, "arbitrary")
        rec = f.f.copy()
        rec["filter_level"] = 64 + np.arange(rec.size).reshape(rec.shape) % 192
        assert same(emu_frame(emulf, f, rec), f.planes)
        f.f["filter_level"][1, 2], f.f["filter_level"][2, 0], f.f["filter_level"][3, 4] = 64, 200, 255
        got = emu_frame(emulf, f)
        assert same(got, vl.orc_frame(f)) and not same(got, f.planes)


def test_emu_simple_leaves_chroma(emulf):
    """the simple filter writes luma only"""
    for is_vp7 in (0, 1):
        f = vl.Frame(510 + is_vp7, 6, 5, is_vp7, 1, 1, "decoder")
        got = emu_frame(emulf, f)
        assert not np.array_equal(got[0], f.planes[0])
        assert np.array_equal(got[1], f.planes[1]) and np.array_equal(got[2], f.planes[2])


def member_call(fn, m, E, I, H, d):
    dir, kind, uv = vl.member_geometry(m)
    p0, p1 = d[0].ctypes.data + 16 * 32 + 16, d[1].ctypes.data + 16 * 32 + 16
    if kind == 2:
        fn(p0, 32, E)
    elif uv:
        fn(p0, p1, 32, E, I, H)
    else:
        fn(p0, 32, E, I, H)


def check_members(ctx, is_vp7, seed):
    """every member through host pointers against the checker: the two 32 x 32 blocks around the edge (what the member may not read or
    write included)"""
    for call in vl.member_calls(seed, is_vp7):
        m, E, I, H, blks = call
        d = blks.copy()
        member_call(getattr(ctx, vl.MEMBERS[m]), m, E, I, H, d)
        assert np.array_equal(d, vl.run_member(cl.oracle(), "orc_vp8_lf_member", is_vp7, call)), (is_vp7, vl.MEMBERS[m], E, I, H)


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
def test_emu_every_member(emulf, is_vp7):
    from ffmpeg_b200._lib import VP8DSPContext
    ctx = VP8DSPContext()
    assert emulf.b200_vp8_dsp_init_loopfilter(C.byref(ctx), is_vp7) == 0
    check_members(ctx, is_vp7, 60 + is_vp7)


def table_words(ctx):
    return np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)


def pointer_pattern(words):
    """the sharing pattern of 70 pointers: 0 for NULL, else the index of the first member holding the same function + 1"""
    first = {}
    return [0 if w == 0 else first.setdefault(int(w), k) + 1 for k, w in enumerate(words)]


def test_emu_init_sets_exactly_the_table(emulf):
    """on top of b200_vp8_dsp_init's context the init sets words 6..15 and nothing else, ten distinct functions per codec, twenty in
    all; after both inits the 70-pointer sharing pattern is the reference's, unmasked"""
    from ffmpeg_b200._lib import VP8DSPContext
    seen = set()
    for is_vp7 in (0, 1):
        ctx = VP8DSPContext()
        assert emulf.b200_vp8_dsp_init(C.byref(ctx), is_vp7) == 0
        w0 = table_words(ctx).copy()
        assert (w0[6:16] == 0).all()
        assert emulf.b200_vp8_dsp_init_loopfilter(C.byref(ctx), is_vp7) == 0
        w1 = table_words(ctx)
        assert list(np.nonzero(w0 != w1)[0]) == list(range(6, 16))
        assert len(set(w1[6:16])) == 10
        seen |= set(w1[6:16])
        pat = np.array(pointer_pattern(w1))

        def reference_pattern():
            out = (C.c_void_p * 70)()
            assert vl.ref().ffref_vp8lf_pointers(is_vp7, out) == 0
            return np.array(pointer_pattern([x or 0 for x in out]))
        with vl.RefCheck() as rc:
            assert rc.same(pat, reference_pattern)
        blank = VP8DSPContext()
        assert emulf.b200_vp8_dsp_init_loopfilter(C.byref(blank), is_vp7) == 0
        wb = table_words(blank)
        assert (wb[6:16] == w1[6:16]).all() and not wb[:6].any() and not wb[16:].any()
    assert len(seen) == 20


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emulf):
    from ffmpeg_b200._lib import VP8DSPContext
    for L in (prodlib, emulf):
        ctx = VP8DSPContext()
        for v in (-1, 2, 8):
            assert L.b200_vp8_dsp_init_loopfilter(C.byref(ctx), v) == EINVAL, v
        assert L.b200_vp8_dsp_init_loopfilter(None, 0) == EINVAL
        assert not table_words(ctx).any()


def test_frame_refusals(prodlib, emulf):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data
    before = emulf.emu_launch_count()
    for L in (prodlib, emulf):
        def call(v7=0, simple=0, kf=0, mbw=2, mbh=2, planes=(p, p + 8192, p + 12288), ls_y=32, ls_uv=16, rec=p + 16384, fstride=2):
            arr = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vp8_loopfilter_frame_device(None, v7, simple, kf, mbw, mbh, arr, ls_y, ls_uv, rec, fstride)
        for k in range(3):
            pl = [p, p + 8192, p + 12288]
            pl[k] = None
            assert call(planes=tuple(pl)) == EINVAL, k
        assert call(planes=None) == EINVAL and call(rec=None) == EINVAL
        for v in (-1, 2, 255):
            assert call(v7=v) == EINVAL and call(simple=v) == EINVAL and call(kf=v) == EINVAL, v
        assert call(mbw=0) == EINVAL and call(mbh=0) == EINVAL and call(mbw=-4) == EINVAL and call(mbh=-1) == EINVAL
        assert call(ls_y=31) == EINVAL and call(ls_uv=15) == EINVAL and call(mbw=3, ls_y=47, ls_uv=24, fstride=3) == EINVAL
        assert call(mbw=3, ls_y=48, ls_uv=23, fstride=3) == EINVAL
        assert call(fstride=1) == EINVAL and call(fstride=-2) == EINVAL and call(mbw=3, ls_y=48, ls_uv=24, fstride=2) == EINVAL
        assert L.b200_vp8_loopfilter_timeouts(None, None) == EINVAL
    assert not b.any()
    assert emulf.emu_launch_count() == before
