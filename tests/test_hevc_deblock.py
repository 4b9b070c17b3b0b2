"""CPU tier for HEVC deblocking (HEVCDSPContext's loop-filter members and b200_hevc_deblock_plane_device, ffmpeg_b200/csrc/hevcdbk.cu):
the checker (oracle/hevcdbk_oracle.c) against the compiled reference (oracle/_ref/libffref_hevcdbk.so) member by member and against the
decoder's CTB-by-CTB order on whole planes, the fixture hashes and their branch coverage, the ctypes mirror, and hevcdbk.cu itself, host
code included, on the stand-in CUDA runtime of tests/cuda_emu (planes, sentinels, ignored grid entries, every member, the refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hevcdbklib as hd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", hd.DEPTHS)
@pytest.mark.parametrize("cls", hd.CLASSES)
def test_checker_members_match_reference(depth, cls):
    """every member (and its _c twin) on decoder-shaped, dense (beta 0..255, tc -255..255, any no_p / no_q byte) and extreme inputs;
    the whole 16 x 16 buffer is compared, so writes outside what the reference writes show"""
    seed = 100 + 13 * depth + hd.CLASSES.index(cls)
    calls = list(hd.member_calls(seed, depth, cls))
    ours = [hd.orc_member(depth, c) for c in calls]
    with hd.RefCheck() as rc:
        assert rc.same(ours, lambda: [hd.ref_member(depth, c) for c in calls])
        assert rc.same(ours, lambda: [hd.ref_member(depth, c, twin=True) for c in calls])


@pytest.mark.parametrize("depth", hd.DEPTHS)
def test_checker_tc_le_0_is_a_no_op(depth):
    """a segment with tc <= 0 is left as it is, luma and chroma (what the plane's per-segment form relies on): the reference with
    that segment's tc at 0 or negative gives the buffer with only the other segment filtered"""
    rng = np.random.default_rng(7 + depth)
    maxv = (1 << depth) - 1
    for fn in range(4):
        for t in (0, -1, -7, -255):
            buf = rng.integers(0, maxv + 1, (16, 16)).astype(hd.sdtype(depth))
            buf[:, 6:10] = maxv // 2 + rng.integers(-3, 4, (16, 4))        # low activity: the luma decision passes
            buf = buf if fn % 2 else np.ascontiguousarray(buf.T)
            for j in range(2):
                tc = [255, 255]
                tc[j] = t
                call = (fn, buf, 255, tc, [0, 0], [0, 0])
                got = hd.orc_member(depth, call)
                lines = slice(hd.EDGE + 4 * j, hd.EDGE + 4 * j + 4)
                same = got[lines, :] if fn % 2 else got[:, lines]
                orig = buf[lines, :] if fn % 2 else buf[:, lines]
                assert np.array_equal(same, orig), (fn, t, j)
                with hd.RefCheck() as rc:
                    assert rc.same(got, lambda: hd.ref_member(depth, call))


@pytest.mark.parametrize("depth", hd.DEPTHS)
@pytest.mark.parametrize("plane", ("luma", "420", "422", "444"))
def test_checker_plane_is_the_decoder_order(depth, plane):
    """the picture-level form (all vertical segments, then all horizontal ones) against the reference's members driven CTB by CTB
    in the decoder's order, at CTB sizes 16, 32 and 64, on decoder-shaped and dense planes"""
    hs, vs = {"luma": (0, 0), "420": (1, 1), "422": (1, 0), "444": (0, 0)}[plane]
    chroma = plane != "luma"
    W, H = (132 >> hs) + (4 if hs else 0), (100 >> vs) + (4 if vs else 0)
    W, H = W - W % 4, H - H % 4
    for log2_ctb in (4, 5, 6):
        for cls in ("decoder", "dense"):
            buf, vg, hg = hd.plane_case(500 + depth + 7 * log2_ctb + len(cls), depth, W, H, chroma, cls, hs, vs, 1 << log2_ctb)
            ours = hd.orc_plane(depth, int(chroma), buf, vg, hg, W, H)
            assert not np.array_equal(ours, buf)
            lw, lh = (log2_ctb - hs, log2_ctb - vs) if chroma else (log2_ctb, log2_ctb)
            with hd.RefCheck() as rc:
                assert rc.same(ours, lambda: hd.ref_plane_ctb(depth, int(chroma), buf, vg, hg, W, H, lw, lh))


def test_fixture_reaches_every_branch_and_matches():
    """the fixture planes: the checker reproduces the stored hashes of the reference's result, and between them the planes reach
    every branch (d >= beta skip, strong, weak with nd_p / nd_q 1 and 2, weak lines skipped by |delta0| >= 10 tc, tc <= 0, chroma)"""
    hs = hd.fixture_hashes()
    assert len(hs) == len(hd.DEPTHS) * 2
    for (depth, chroma), h in hs.items():
        (buf, vg, hg), W, H = hd.fixture_case(depth, int(chroma))
        assert hd.digest(hd.orc_plane(depth, int(chroma), buf, vg, hg, W, H)) == h, (depth, chroma)
        cnt = hd.branch_counts(depth, int(chroma), buf, vg, hg, W, H)
        need = ("tc_le_0", "chroma_filtered") if chroma else ("skip_d_ge_beta", "strong", "weak_ndp1", "weak_ndp2", "weak_ndq1",
                                                              "weak_ndq2", "weak_line_skipped", "tc_le_0")
        assert all(cnt[k] > 0 for k in need), (depth, chroma, cnt)


def test_fixture_is_the_reference_result():
    if not hd.have_ref():
        pytest.skip("the reference is not built here; test_fixture_reaches_every_branch_and_matches checks the stored hashes")
    for (depth, chroma), h in hd.fixture_hashes().items():
        (buf, vg, hg), W, H = hd.fixture_case(depth, int(chroma))
        got = hd.ref_plane_ctb(depth, int(chroma), buf, vg, hg, W, H, 5 - chroma, 5 - chroma)
        assert hd.digest(got) == h


def test_ctypes_mirror():
    from ffmpeg_b200._lib import HevcDbkSeg
    from ffmpeg_b200 import hevcdsp
    assert C.sizeof(HevcDbkSeg) == hevcdsp.DBK_DTYPE.itemsize == 4
    for name, _ in HevcDbkSeg._fields_:
        assert getattr(HevcDbkSeg, name).offset == hevcdsp.DBK_DTYPE.fields[name][1], name


# ---------------------------------------------------------------- hevcdbk.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emudbk():
    """libemuhevcdbk.so: hevcdbk.cu with its host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The kernel uses
    shared memory, __syncthreads and __shfl_sync, so it runs an OS thread per CUDA thread of a block (emu.h's block launch), with
    __shfl_sync built on that launch's warp exchange."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("hevcdbk.cu", "tx_pfa.cu"):                          # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "hevcdbk.cu":
            assert t.count("extern __shared__ uint16_t dbk_tile[];") == 1 and t.count("emu_cfg_launch(0, [&] { hevc_dbk_kernel<") == 4
            t = t.replace("extern __shared__ uint16_t dbk_tile[];", "uint16_t *dbk_tile = (uint16_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_dbk_kernel<", "emu_cfg_launch(2, [&] { hevc_dbk_kernel<")
            t = t.replace('#include "common.h"', '#include "common.h"\nstatic inline int __shfl_sync(unsigned, int v, int l) '
                                                 '{ return (int)emu_warp_xchg((unsigned)v, l); }', 1)
        assert "<<<" not in t
        p = os.path.join(gen, "dbk_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuhevcdbk.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_hevc_dsp_init_deblock.argtypes = [C.c_void_p, C.c_int]
    L.b200_hevc_deblock_plane_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p,
                                                 C.c_int64, C.c_void_p, C.c_int64]
    L.emu_launch_count.restype = C.c_uint64
    L.b200_last_error.restype = C.c_char_p
    return L


def emu_plane(L, depth, chroma, buf, vg, hg, W, H):
    d, v0, h0 = buf.copy(), vg.copy(), hg.copy()
    assert L.b200_hevc_deblock_plane_device(None, depth, chroma, hd._plane_ptr(d), d.strides[0], W, H, v0.ctypes.data, vg.shape[1],
                                            h0.ctypes.data, hg.shape[1]) == 0
    assert np.array_equal(v0, vg) and np.array_equal(h0, hg)
    return d


@pytest.mark.parametrize("depth", hd.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_emu_plane_vs_checker_and_fixture(emudbk, depth, chroma):
    """the fixture plane (W, H = 4 mod 8, more than one tile each way) through the library's entry: equal to the checker over the
    whole buffer (sentinels around the plane unchanged; the non-zero entries at x = 0 / y = 0 and the garbage in the grid padding
    ignored) and to the reference's hash"""
    (buf, vg, hg), W, H = hd.fixture_case(depth, chroma)
    got = emu_plane(emudbk, depth, chroma, buf, vg, hg, W, H)
    assert np.array_equal(got, hd.orc_plane(depth, chroma, buf, vg, hg, W, H))
    assert hd.digest(got) == hd.fixture_hashes()[(depth, bool(chroma))]
    inner = np.zeros(got.shape, bool)
    inner[hd.MARGIN:hd.MARGIN + H, hd.MARGIN:hd.MARGIN + W] = True
    assert np.array_equal(got[~inner], buf[~inner])


@pytest.mark.parametrize("cls", ("dense", "extreme"))
def test_emu_plane_classes(emudbk, cls):
    """dense (random beta / tc / flags, any flag bits) and extreme (0 / maximum samples, beta = tc = 255) planes at 8 and 10 bit,
    luma and chroma, against the checker"""
    for depth in (8, 10):
        for chroma in (0, 1):
            W, H = (140, 36) if chroma else (132, 44)
            buf, vg, hg = hd.plane_case(40 + depth + chroma + len(cls), depth, W, H, bool(chroma), cls)
            assert np.array_equal(emu_plane(emudbk, depth, chroma, buf, vg, hg, W, H), hd.orc_plane(depth, chroma, buf, vg, hg, W, H))


def test_emu_every_member(emudbk):
    """all eight member pointers at every depth, called through the context with host pointers, against the checker on every class;
    each _c pointer is its plain twin"""
    from ffmpeg_b200._lib import HEVCDSPContext
    for depth in hd.DEPTHS:
        ctx = HEVCDSPContext()
        assert emudbk.b200_hevc_dsp_init_deblock(C.byref(ctx), depth) == 0
        for n in ("h_loop_filter_luma", "v_loop_filter_luma", "h_loop_filter_chroma", "v_loop_filter_chroma"):
            assert getattr(ctx, "hevc_" + n) and getattr(ctx, "hevc_" + n) == getattr(ctx, "hevc_" + n + "_c")
        for cls in hd.CLASSES:
            for call in hd.member_calls(80 + depth + len(cls), depth, cls):
                assert np.array_equal(hd.ctx_member(ctx, call), hd.orc_member(depth, call)), (depth, cls, call[0], call[2:])


def test_emu_member_tc_le_0_launches_nothing(emudbk):
    from ffmpeg_b200._lib import HEVCDSPContext
    ctx = HEVCDSPContext()
    assert emudbk.b200_hevc_dsp_init_deblock(C.byref(ctx), 10) == 0
    before = emudbk.emu_launch_count()
    buf = np.arange(256, dtype=np.uint16).reshape(16, 16)
    for fn in range(4):
        assert np.array_equal(hd.ctx_member(ctx, (fn, buf, 64, [0, -3], [0, 0], [0, 0])), buf)
    assert emudbk.emu_launch_count() == before


def test_emu_init_sets_exactly_the_deblocking_members(emudbk):
    """the eight loop-filter pointers are set, every other member of a filled context stays as it was"""
    from ffmpeg_b200._lib import HEVCDSPContext
    ctx = HEVCDSPContext()
    C.memset(C.addressof(ctx), 0x11, C.sizeof(ctx))
    before = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64).copy()
    assert emudbk.b200_hevc_dsp_init_deblock(C.byref(ctx), 12) == 0
    words = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
    dbk = np.zeros(len(words), bool)
    dbk[-8:] = True
    assert (words[dbk] != before[dbk]).all() and np.array_equal(words[~dbk], before[~dbk])


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emudbk):
    from ffmpeg_b200._lib import HEVCDSPContext
    for L in (prodlib, emudbk):
        ctx = HEVCDSPContext()
        for depth in (0, 7, 11, 13, 14, 16):
            assert L.b200_hevc_dsp_init_deblock(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_hevc_dsp_init_deblock(None, 8) == EINVAL
        assert not any(bytes(ctx))


def test_plane_refusals(prodlib, emudbk):
    """every B200_EINVAL case launches nothing and writes nothing"""
    pix = np.zeros(64 * 64 * 2 + 64, np.uint8)
    base = (pix.ctypes.data + 63) & ~63
    g = np.full(4096, 0x3F, np.uint8)
    grid = g.ctypes.data
    before = emudbk.emu_launch_count()
    for L in (prodlib, emudbk):
        def call(depth=8, chroma=0, p=base, stride=64, W=32, H=32, v=grid, vs=4, h=grid, hs=8):
            return L.b200_hevc_deblock_plane_device(None, depth, chroma, p, stride, W, H, v, vs, h, hs)
        for k in ("p", "v", "h"):
            assert call(**{k: None}) == EINVAL, k
        for depth in (0, 7, 11, 13, 16):
            assert call(depth=depth) == EINVAL, depth
        for chroma in (-1, 2, 255):
            assert call(chroma=chroma) == EINVAL, chroma
        for W, H in ((0, 32), (2, 32), (30, 32), (33, 32), (32, 0), (32, 3), (32, 30), (-8, 32), (32, -8)):
            assert call(W=W, H=H) == EINVAL, (W, H)
        assert call(stride=31) == EINVAL and call(stride=-64) == EINVAL and call(stride=0) == EINVAL
        assert call(depth=10, stride=63) == EINVAL and call(depth=10, stride=65) == EINVAL and call(depth=10, p=base + 1, stride=64) == EINVAL
        assert call(vs=3) == EINVAL and call(hs=7) == EINVAL and call(W=36, vs=4) == EINVAL and call(vs=-1) == EINVAL
    assert not pix.any() and (g == 0x3F).all()
    assert emudbk.emu_launch_count() == before
