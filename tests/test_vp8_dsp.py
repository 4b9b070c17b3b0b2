"""CPU tier for VP8 / VP7 motion compensation and residual (VP8DSPContext's MC tables and residual members, ffmpeg_b200/csrc/vp8mc.cu
and vp8idct.cu): the checker (oracle/vp8dsp_oracle.c) against the compiled reference (oracle/_ref/libffref_vp8dsp.so) member by member
and on the decoder's two frame sequences, the filter tables, the fixture hashes, the layout marker, the ctypes mirrors, and both .cu
files, host code included, on the stand-in CUDA runtime of tests/cuda_emu (the frame entries, sentinels, every table entry, the member
pattern and the refusals)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vp8dsplib as v8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL = -22


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("bilinear", (0, 1), ids=("epel", "bilinear"))
@pytest.mark.parametrize("cls", (0, 1), ids=("noise", "extremes"))
def test_checker_mc_members_match_reference(bilinear, cls):
    """every non-NULL entry of both tables with every phase it takes (all 7 at every epel position, the 4-tap ones with even phases
    included), h over 1..2w"""
    seed = 100 + 7 * bilinear + cls
    calls = list(v8.mc_calls(seed, bilinear))
    assert {(c[2], c[3], c[5]) for c in calls if c[3]} >= {(v, h, m) for (_, v, h) in v8.positions(bilinear) if h for m in range(1 - bilinear, 8)}
    ours = v8.run_members(cl.oracle(), "orc", seed, bilinear, cls)
    with v8.RefCheck() as rc:
        assert rc.same(ours, lambda: v8.run_members(v8.ref(), "ffref", seed, bilinear, cls))


def test_sixtap_reaches_both_clip_bounds():
    """on the extremes picture the 6-tap sums leave 0..255 on both sides in the horizontal pass and in the vertical pass over the
    clipped intermediates, so a missing clip in either shows in the member tests"""
    pic, _ = v8.member_case(101, 1)
    F = v8.subpel_filters(cl.oracle(), "orc_vp8_subpel_filters").astype(np.int64) * np.array([1, -1, 1, 1, -1, 1])
    p = pic.astype(np.int64)
    for m in (2, 4, 6):
        hs = (sum(F[m - 1][k] * p[:, k:p.shape[1] - 5 + k] for k in range(6)) + 64) >> 7
        assert hs.min() < 0 and hs.max() > 255, (m, hs.min(), hs.max())
        t = hs.clip(0, 255)
        vs = (sum(F[m - 1][k] * t[k:t.shape[0] - 5 + k] for k in range(6)) + 64) >> 7
        assert vs.min() < 0 and vs.max() > 255, (m, vs.min(), vs.max())


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
@pytest.mark.parametrize("kind", ("decoder", "dense", "extreme"))
def test_checker_residual_members_match_reference(is_vp7, kind):
    seed = 300 + 10 * is_vp7 + ("decoder", "dense", "extreme").index(kind)
    ours = v8.residual_member_runs(cl.oracle(), "orc", seed, is_vp7, kind)
    with v8.RefCheck() as rc:
        assert rc.same(ours, lambda: v8.residual_member_runs(v8.ref(), "ffref", seed, is_vp7, kind))


@pytest.mark.parametrize("bilinear", (0, 1), ids=("epel", "bilinear"))
@pytest.mark.parametrize("cls", (0, 1), ids=("noise", "extremes"))
def test_checker_mc_frame_matches_decoder_sequence(bilinear, cls):
    """the checker's clamped windows against the reference driver's edge test + emulated_edge_mc windows + member calls: every
    partitioning, windows up to 80 samples outside the plane"""
    refs, ops, dst = v8.mc_case(400 + 2 * bilinear + cls, 11, 7, cls=cls)
    ours = v8.orc_mc_frame(bilinear, 11, 7, refs, ops, dst)
    assert not np.array_equal(ours[0], dst[0]) and not np.array_equal(ours[2], dst[2])
    with v8.RefCheck() as rc:
        assert rc.same(ours, lambda: v8.ref_mc_frame(bilinear, 11, 7, refs, ops, dst))


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
@pytest.mark.parametrize("kind", ("decoder", "dense", "extreme"))
def test_checker_residual_frame_matches_decoder_sequence(is_vp7, kind):
    """the WHT and idct_mb with its dc_add4y / dc_add4uv branches, early break and goto"""
    rng = np.random.default_rng(500 + is_vp7)
    ops, coef = v8.residual_case(510 + 3 * is_vp7 + len(kind), 10, 6, is_vp7, kind)
    dst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v8.dst_planes(10, 6)]
    ours = v8.orc_residual_frame(is_vp7, ops, coef, dst)
    with v8.RefCheck() as rc:
        assert rc.same(ours, lambda: v8.ref_residual_frame(is_vp7, ops, coef, dst))


def test_context_layout_matches_reference():
    """oracle/ref/ref_vp8dsp.c asserts at compile time that B200VP8DSPContext has VP8DSPContext's size, member offsets and types"""
    if not v8.have_ref():
        pytest.skip("oracle/_ref/libffref_vp8dsp.so not built")
    marker = C.c_char_p.in_dll(v8.ref(), "ffref_vp8dsp_layout_check")
    assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200VP8DSPContext matches")


def pointer_pattern(words):
    """the sharing pattern of 70 pointers: 0 for NULL, else the index of the first member holding the same function + 1"""
    first = {}
    return [0 if w == 0 else first.setdefault(int(w), k) + 1 for k, w in enumerate(words)]


def reference_pattern(is_vp7):
    """the reference's pattern with the ten loop-filter members NULL (not built here); from the reference where it is built"""
    if v8.have_ref():
        out = (C.c_void_p * 70)()
        assert v8.ref().ffref_vp8_pointers(is_vp7, out) == 0
        words = [x or 0 for x in out]
        words[6:16] = [0] * 10
        return pointer_pattern(words)
    return None


def kernel_filters():
    """the rows of vp8mc.cu's c_vp8_filters, parsed from the source: [3][8][6]"""
    txt = open(os.path.join(ROOT, "ffmpeg_b200", "csrc", "vp8mc.cu")).read()
    body = txt[txt.index("c_vp8_filters[3][8][6] = {"):]
    body = body[:body.index("};")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{([-0-9, ]+)\}", body)]
    return np.array(rows, np.int64).reshape(3, 8, 6)


def test_filter_tables():
    """the kernel's banks against the checker's subpel_filters (against the reference's through the member tests): 6-tap rows with
    the reference's signs, 4-tap rows with the outer taps zeroed, phase 0 the identity; the bilinear bank is the 6-tap form of
    ((8 - m) s0 + m s1 + 4) >> 3, proven for every pair of samples, and its results never leave 0..255"""
    K = kernel_filters()
    F = v8.subpel_filters(cl.oracle(), "orc_vp8_subpel_filters").astype(np.int64) * np.array([1, -1, 1, 1, -1, 1])
    assert (F.sum(axis=1) == 128).all()
    assert list(K[0][0]) == list(K[1][0]) == list(K[2][0]) == [0, 0, 128, 0, 0, 0]
    assert np.array_equal(K[0][1:], F)
    four = F.copy()
    four[:, 0] = four[:, 5] = 0
    assert np.array_equal(K[1][1:], four)
    assert (F[0::2, 0] == 0).all() and (F[0::2, 5] == 0).all()          # odd phases: the 6-tap row is the 4-tap row
    a, b = np.meshgrid(np.arange(256), np.arange(256))
    for m in range(8):
        assert list(K[2][m]) == [0, 0, 128 - 16 * m, 16 * m, 0, 0]
        got = (K[2][m][2] * a + K[2][m][3] * b + 64) >> 7
        assert np.array_equal(got, ((8 - m) * a + m * b + 4) >> 3)
        assert got.min() >= 0 and got.max() <= 255


def test_checker_reproduces_fixture():
    hs = v8.fixture_hashes()
    assert sorted(hs) == sorted(v8.FIXTURE_CASES)
    for (is_vp7, bil), h in hs.items():
        refs, ops, dst, rops, coef = v8.fixture_case(is_vp7, bil)
        planes = v8.orc_residual_frame(is_vp7, rops, coef, v8.orc_mc_frame(bil, 12, 9, refs, ops, dst))
        assert v8.digest(planes) == h, (is_vp7, bil)


def test_ctypes_mirrors():
    from ffmpeg_b200._lib import VP8DSPContext, Vp8McOp, Vp8McRef, Vp8ResidualOp
    from ffmpeg_b200 import vp8dsp
    assert C.sizeof(Vp8McOp) == vp8dsp.MC_DTYPE.itemsize == 24 and C.sizeof(Vp8McRef) == 40
    assert C.sizeof(Vp8ResidualOp) == vp8dsp.RES_DTYPE.itemsize == 48
    for name, _ in Vp8McOp._fields_:
        assert getattr(Vp8McOp, name).offset == vp8dsp.MC_DTYPE.fields[name][1], name
    for name, _ in Vp8ResidualOp._fields_:
        assert getattr(Vp8ResidualOp, name).offset == vp8dsp.RES_DTYPE.fields[name][1], name
    assert C.sizeof(VP8DSPContext) == 70 * 8 and VP8DSPContext.put_vp8_epel_pixels_tab.offset == 16 * 8
    assert VP8DSPContext.put_vp8_bilinear_pixels_tab.offset == 43 * 8


# ---------------------------------------------------------------- vp8mc.cu / vp8idct.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emuvp8():
    """libemuvp8.so: vp8mc.cu and vp8idct.cu with their host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The MC
    kernel uses shared memory and __syncwarp, so it runs an OS thread per CUDA thread of a block and __syncwarp becomes the warp's
    barrier; the residual kernels have no collective and run thread after thread."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vp8mc.cu", "vp8idct.cu", "tx_pfa.cu"):                 # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vp8mc.cu":
            assert t.count("extern __shared__ uint32_t vp8_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { vp8_mc_kernel(") == 1
            t = t.replace("extern __shared__ uint32_t vp8_smem[];", "uint32_t *vp8_smem = (uint32_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { vp8_mc_kernel(", "emu_cfg_launch(2, [&] { vp8_mc_kernel(")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, "vp8_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuvp8.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_vp8_dsp_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp8_mc_frame_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                           C.c_ssize_t, C.c_ssize_t]
    L.b200_vp8_residual_frame_device.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t]
    L.emu_launch_count.restype = C.c_uint64
    return L


def emu_mc(L, bilinear, mbw, mbh, refs, ops, dst):
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    assert L.b200_vp8_mc_frame_device(None, bilinear, mbw, mbh, len(refs), C.cast(v8.ref_array(refs), C.c_void_p), len(ops), ops.ctypes.data,
                                      planes, d[0].strides[0], d[1].strides[0]) == 0
    return d


def emu_residual(L, is_vp7, ops, coef, dst):
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    assert L.b200_vp8_residual_frame_device(None, is_vp7, len(ops), ops.ctypes.data, coef.ctypes.data, planes, d[0].strides[0],
                                            d[1].strides[0]) == 0
    return d


@pytest.mark.parametrize("is_vp7,bilinear", v8.FIXTURE_CASES, ids=("vp8-epel", "vp8-bilinear", "vp7-epel", "vp7-bilinear"))
def test_emu_fixture_frames(emuvp8, is_vp7, bilinear):
    """the fixture frames through both entries: equal to the checker after each, the sentinels of the intra MBs and of the padding
    right of and below every plane unchanged, and the reference's hash at the end"""
    refs, ops, dst, rops, coef = v8.fixture_case(is_vp7, bilinear)
    got = emu_mc(emuvp8, bilinear, 12, 9, refs, ops, dst)
    exp = v8.orc_mc_frame(bilinear, 12, 9, refs, ops, dst)
    assert all(np.array_equal(a, b) for a, b in zip(got, exp))
    for p, s in zip(got, (16, 8, 8)):
        assert (p[9 * s:] == v8.SENTINEL).all() and (p[:, 12 * s:] == v8.SENTINEL).all()
    assert (got[0][:144, :192] == v8.SENTINEL).sum() >= 256 * 0.5 * (108 - len(set(zip(ops["dst_x"] // 16, ops["dst_y"] // 16))))
    got = emu_residual(emuvp8, is_vp7, rops, coef, got)
    assert all(np.array_equal(a, b) for a, b in zip(got, v8.orc_residual_frame(is_vp7, rops, coef, exp)))
    assert v8.digest(got) == v8.fixture_hashes()[(is_vp7, bilinear)]


def test_emu_large_frames(emuvp8):
    """more than 8000 ops in one call of each entry (an 80 x 40 MB frame on the extremes pictures; dense residual coefficients)"""
    refs, ops, dst = v8.mc_case(61, 80, 40, cls=1, intra=0.0)
    assert len(ops) > 8000
    got = emu_mc(emuvp8, 0, 80, 40, refs, ops, dst)
    assert all(np.array_equal(a, b) for a, b in zip(got, v8.orc_mc_frame(0, 80, 40, refs, ops, dst)))
    rops, coef = v8.residual_case(62, 120, 70, 0, "dense", skip=0.0)
    assert len(rops) > 8000
    got2 = emu_residual(emuvp8, 0, rops, coef, [np.zeros((16 * 70, 16 * 120), np.uint8)] + [np.zeros((8 * 70, 8 * 120), np.uint8)] * 2)
    exp2 = v8.orc_residual_frame(0, rops, coef, [np.zeros((16 * 70, 16 * 120), np.uint8)] + [np.zeros((8 * 70, 8 * 120), np.uint8)] * 2)
    assert all(np.array_equal(a, b) for a, b in zip(got2, exp2))


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
@pytest.mark.parametrize("kind", ("decoder", "dense", "extreme"))
def test_emu_residual_frame_vs_checker(emuvp8, is_vp7, kind):
    rng = np.random.default_rng(70 + is_vp7)
    ops, coef = v8.residual_case(71 + 3 * is_vp7 + len(kind), 10, 6, is_vp7, kind)
    dst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v8.dst_planes(10, 6)]
    assert all(np.array_equal(a, b) for a, b in zip(emu_residual(emuvp8, is_vp7, ops, coef, dst), v8.orc_residual_frame(is_vp7, ops, coef, dst)))


def test_emu_invalid_ops_write_nothing(emuvp8):
    """undefined plane classes and widths, h outside 1..16, phases above 7, a reference index >= nrefs, 16-wide epel ops with an odd
    phase, a dst_x not a multiple of 4, blocks not inside the plane; residual ops with a negative MB position or an unaligned coef_off:
    nothing written, while the valid ops of the same call are"""
    refs, ops, dst = v8.mc_case(81, 6, 5, intra=0.0)
    bad = ops[:16].copy()
    bad["plane"][0], bad["w"][1], bad["w"][2], bad["h"][3], bad["h"][4] = 2, 12, 32, 0, 17
    bad["mx"][5], bad["my"][6], bad["ref"][7] = 8, 255, 3
    bad["w"][8], bad["h"][8], bad["mx"][8], bad["plane"][8] = 16, 16, 3, 0
    bad["dst_x"][9] += 2
    bad["dst_x"][10], bad["dst_y"][11], bad["dst_x"][12], bad["dst_y"][13] = -4, -1, 96, 80
    bad["dst_x"][14], bad["w"][14], bad["plane"][14] = 48 - 4, 8, 1
    bad["dst_y"][15], bad["h"][15], bad["plane"][15] = 76, 8, 0
    for bil in (0, 1):
        n = 16 if not bil else 15
        sel = bad if not bil else np.delete(bad, 8)
        assert all(np.array_equal(a, b) for a, b in zip(emu_mc(emuvp8, bil, 6, 5, refs, sel[:n], dst), dst)), bil
        assert all(np.array_equal(a, b) for a, b in zip(v8.orc_mc_frame(bil, 6, 5, refs, sel[:n], dst), dst))
    mixed = np.concatenate([bad, ops[16:]])
    got = emu_mc(emuvp8, 0, 6, 5, refs, mixed, dst)
    assert all(np.array_equal(a, b) for a, b in zip(got, v8.orc_mc_frame(0, 6, 5, refs, mixed, dst))) and not np.array_equal(got[0], dst[0])
    # the 16-wide odd-phase op is valid with the bilinear table
    odd = bad[8:9]
    assert not np.array_equal(emu_mc(emuvp8, 1, 6, 5, refs, odd, dst)[0], dst[0])
    rops, coef = v8.residual_case(82, 6, 5, 0, "dense", skip=0.0)
    rbad = rops[:4].copy()
    rbad["mb_x"][0], rbad["mb_y"][1], rbad["coef_off"][2], rbad["coef_off"][3] = -1, -2, 4, -400
    rng = np.random.default_rng(83)
    rdst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v8.dst_planes(6, 5)]
    assert all(np.array_equal(a, b) for a, b in zip(emu_residual(emuvp8, 0, rbad, coef, rdst), rdst))
    rmixed = np.concatenate([rbad, rops[4:]])
    got = emu_residual(emuvp8, 0, rmixed, coef, rdst)
    assert all(np.array_equal(a, b) for a, b in zip(got, v8.orc_residual_frame(0, rmixed, coef, rdst))) and not np.array_equal(got[0], rdst[0])


def test_emu_every_table_entry(emuvp8):
    """every MC entry of both tables through host pointers against the checker (every third call, which still takes every entry and
    phase), every residual member of both contexts, and out-of-domain member arguments writing nothing"""
    from ffmpeg_b200._lib import VP8DSPContext
    from test_vp8_dsp_gpu import check_mc_members, check_residual_members, run_ctx_mc
    for is_vp7 in (0, 1):
        ctx = VP8DSPContext()
        assert emuvp8.b200_vp8_dsp_init(C.byref(ctx), is_vp7) == 0
        for bil in (0, 1):
            check_mc_members(ctx, bil, 90 + is_vp7 + 2 * bil, is_vp7, stride=3)
        check_residual_members(ctx, is_vp7, 95 + is_vp7)
    pic, dst0 = v8.member_case(1, 0)
    for call in ((0, 8, 2, 2, 0, 3, 3), (0, 8, 2, 2, 17, 3, 3), (0, 8, 2, 0, 8, 3, 0), (0, 4, 1, 1, 4, 8, 3), (1, 4, 1, 1, 4, 8, 3),
                 (0, 8, 0, 2, 4, 0, 1)):
        assert np.array_equal(run_ctx_mc(ctx, call, pic, dst0), dst0), call


def test_emu_member_pattern(emuvp8):
    """the residual members and both MC tables filled, the loop-filter members NULL, the epel [0][1][*] / [0][*][1] NULL; functions
    shared as in the reference (the full-pel entry of a size by both tables, the bilinear positions that filter in the same directions),
    the residual members different for VP7 and VP8, the MC ones the same"""
    from ffmpeg_b200._lib import VP8DSPContext
    words = {}
    for is_vp7 in (0, 1):
        ctx = VP8DSPContext()
        assert emuvp8.b200_vp8_dsp_init(C.byref(ctx), is_vp7) == 0
        w = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
        words[is_vp7] = w
        assert (w[:6] != 0).all() and (w[6:16] == 0).all()
        epel = w[16:43].reshape(3, 3, 3)
        assert (epel[0, 1, :] == 0).all() and (epel[0, :, 1] == 0).all() and (np.delete(w[16:], [1, 3, 4, 5, 7]) != 0).all()
        assert len(set(w[:6])) == 6 and len(set(int(x) for x in w[16:] if x)) == 22 + 9
        pat = pointer_pattern(w)
        ref = reference_pattern(is_vp7)
        if ref is not None:
            assert pat == ref
        with v8.RefCheck() as rc:
            assert rc.same(np.array(pat), lambda: np.array(reference_pattern(is_vp7)))
    assert not set(words[0][:6]) & set(words[1][:6]) and np.array_equal(words[0][16:], words[1][16:])


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emuvp8):
    from ffmpeg_b200._lib import VP8DSPContext
    for L in (prodlib, emuvp8):
        ctx = VP8DSPContext()
        for v in (-1, 2, 8):
            assert L.b200_vp8_dsp_init(C.byref(ctx), v) == EINVAL, v
        assert L.b200_vp8_dsp_init(None, 0) == EINVAL


def test_frame_refusals(prodlib, emuvp8):
    """every B200_EINVAL case of both entries launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    from ffmpeg_b200._lib import Vp8McRef
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data
    ops = np.zeros(1, v8.MC_DTYPE)
    ops["w"] = ops["h"] = 4
    rops = np.zeros(1, v8.RES_DTYPE)
    rops["nnz"] = 2
    rops["flags"] = 1
    before = emuvp8.emu_launch_count()
    for L in (prodlib, emuvp8):
        def mc(bil=0, mbw=2, mbh=2, nrefs=1, n=1, ops=ops.ctypes.data, refs=True, planes=(p + 1024, p + 4096, p + 8192), ls_y=64, ls_uv=32,
               ref_planes=(p + 16384, p + 20480, p + 24576)):
            arr = (Vp8McRef * 3)(*[Vp8McRef(*ref_planes, 64, 32)] * 3)
            dp = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vp8_mc_frame_device(None, bil, mbw, mbh, nrefs, C.cast(arr, C.c_void_p) if refs else None, n, ops, dp, ls_y, ls_uv)
        assert mc(n=0) == 0 and mc(n=0, ops=None, refs=False, planes=None) == 0
        assert mc(n=-1) == EINVAL and mc(nrefs=0) == EINVAL and mc(nrefs=4) == EINVAL and mc(nrefs=-1) == EINVAL
        assert mc(mbw=0) == EINVAL and mc(mbh=0) == EINVAL and mc(mbw=-3) == EINVAL
        assert mc(ops=None) == EINVAL and mc(refs=False) == EINVAL and mc(planes=None) == EINVAL and mc(ops=ops.ctypes.data + 2) == EINVAL
        for k in range(3):
            pl = [p + 1024, p + 4096, p + 8192]
            pl[k] = 0
            assert mc(planes=tuple(pl)) == EINVAL, k
            pl[k] = [p + 1025, p + 4098, p + 8195][k]
            assert mc(planes=tuple(pl)) == EINVAL, k
            rp = [p + 16384, p + 20480, p + 24576]
            rp[k] = 0
            assert mc(ref_planes=tuple(rp)) == EINVAL, k
        assert mc(ls_y=66) == EINVAL and mc(ls_uv=33) == EINVAL

        def res(v7=0, n=1, ops=rops.ctypes.data, coef=p + 32768, planes=(p + 1024, p + 4096, p + 8192), ls_y=64, ls_uv=32):
            dp = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vp8_residual_frame_device(None, v7, n, ops, coef, dp, ls_y, ls_uv)
        assert res(n=0) == 0 and res(n=0, ops=None, coef=None, planes=None) == 0
        assert res(n=-1) == EINVAL and res(v7=2) == EINVAL and res(v7=-1) == EINVAL
        assert res(ops=None) == EINVAL and res(coef=None) == EINVAL and res(planes=None) == EINVAL
        assert res(ops=rops.ctypes.data + 4) == EINVAL and res(coef=p + 32776) == EINVAL
        assert res(planes=(p + 1026, p + 4096, p + 8192)) == EINVAL and res(planes=(p + 1024, 0, p + 8192)) == EINVAL
        assert res(ls_y=62) == EINVAL and res(ls_uv=30) == EINVAL
    assert not b.any()
    assert emuvp8.emu_launch_count() == before
