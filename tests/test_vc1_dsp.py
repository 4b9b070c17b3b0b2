"""CPU tier for VC-1 motion compensation and inverse transforms (VC1DSPContext's MC tables and transforms, ffmpeg_b200/csrc/vc1mc.cu and
vc1idct.cu): the checker (oracle/vc1dsp_oracle.c) against the compiled reference (oracle/_ref/libffref_vc1dsp.so) member by member and on
the decoder's two frame sequences, the fixture hashes, the layout marker, the ctypes mirrors, and both .cu files, host code included, on
the stand-in CUDA runtime of tests/cuda_emu (the frame entries, the poisoned padding, every table entry and the refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vc1dsplib as v1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------- the checker against the reference
def test_checker_mc_members_match_reference():
    """every mspel entry (both sizes, all 16 dxy, put and avg, rnd 0 and 1) and both chroma widths at every (x, y), put and avg"""
    ours = v1.run_members(cl.oracle(), "orc", 11)
    with v1.RefCheck() as rc:
        assert rc.same(ours, lambda: v1.run_members(v1.ref(), "ffref", 11))


@pytest.mark.parametrize("kind", ("decoder", "dense", "extreme"))
def test_checker_transforms_match_reference(kind):
    """all eight transforms: dest and what each leaves in block, int16 extremes included"""
    ours = v1.run_itx(cl.oracle(), "orc", 20 + len(kind), kind)
    with v1.RefCheck() as rc:
        assert rc.same(ours, lambda: v1.run_itx(v1.ref(), "ffref", 20 + len(kind), kind))


def test_transforms_reach_int16_truncation():
    """on the extremes the 8-point first pass leaves int16 in both directions, so the reference's truncation matters"""
    rng = np.random.default_rng(5)
    b = v1.coef_blocks(rng, 64, "extreme").astype(np.int64)
    e0, e1 = 12 * (b[:, 0] + b[:, 4]) + 4, 16 * b[:, 1] + 15 * b[:, 3] + 9 * b[:, 5] + 4 * b[:, 7]
    first = (e0 + 16 * b[:, 2] + 6 * b[:, 6] + e1) >> 3
    assert (first > 32767).any() and (first < -32768).any()


@pytest.mark.parametrize("name", [c[0] for c in v1.FIXTURE_CASES])
def test_checker_frames_match_decoder_sequence(name):
    """the checker's MC and residual frames against the reference driver's edge test + emulated_edge_mc windows + range reduction +
    LUTs + member calls, and vc1_decode_p_block's dispatch"""
    mbw, mbh, H, V, refs, ops, dst, rops, coef = v1.fixture_case(name)
    mc = v1.orc_mc_frame(mbw, mbh, H, V, refs, ops, dst)
    res = v1.orc_residual_frame(mbw, mbh, rops, coef, mc)
    assert not np.array_equal(mc[0], dst[0]) and not np.array_equal(res[0], mc[0])
    with v1.RefCheck() as rc:
        assert rc.same(mc, lambda: v1.ref_mc_frame(mbw, mbh, H, V, refs, ops, dst))
        assert rc.same(res, lambda: v1.ref_residual_frame(mbw, mbh, rops, coef, mc))


def test_checker_reproduces_fixture():
    hs = v1.fixture_hashes()
    assert sorted(hs) == sorted(c[0] for c in v1.FIXTURE_CASES)
    for name, h in hs.items():
        mbw, mbh, H, V, refs, ops, dst, rops, coef = v1.fixture_case(name)
        planes = v1.orc_residual_frame(mbw, mbh, rops, coef, v1.orc_mc_frame(mbw, mbh, H, V, refs, ops, dst))
        assert v1.digest(planes) == h, name


def test_fixture_reads_poison_and_edges():
    """the fixture frames take both sides of every edge test: windows copied and planes read directly, with the poisoned padding
    inside the MB grid, so clamping where the decoder reads the plane (or the reverse) changes the result"""
    fired = direct = 0
    for name in ("p-mspel-rnd0", "p-hpel-rnd1"):
        mbw, mbh, H, V, refs, ops, dst, rops, coef = v1.fixture_case(name)
        assert H < 16 * mbw and V < 16 * mbh
        for o in ops:
            if o["kind"] == v1.MC_1MV:
                ms = int(o["flags"] & v1.MSPEL)
                s = o["src"][0]
                x, y, mx, my = int(s["x"]), int(s["y"]), int(s["mx"]), int(s["my"])
                f = (x - ms) % (1 << 32) > H - mx - 16 - 3 * ms or (y - 1) % (1 << 32) > V - my - 19
                fired, direct = fired + f, direct + (not f)
    assert fired > 10 and direct > 30


def test_context_layout_matches_reference():
    """oracle/ref/ref_vc1dsp.c asserts at compile time that B200VC1DSPContext has VC1DSPContext's size, member offsets and types"""
    if not v1.have_ref():
        pytest.skip("oracle/_ref/libffref_vc1dsp.so not built")
    marker = C.c_char_p.in_dll(v1.ref(), "ffref_vc1dsp_layout_check")
    assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200VC1DSPContext matches")


def test_ctypes_mirrors():
    from ffmpeg_b200._lib import VC1DSPContext, Vc1McOp, Vc1McRef, Vc1McSrc, Vc1ResidualOp
    from ffmpeg_b200 import vc1dsp
    assert C.sizeof(Vc1McOp) == vc1dsp.MC_DTYPE.itemsize == 40 and C.sizeof(Vc1McSrc) == 16 and C.sizeof(Vc1McRef) == 1080
    assert C.sizeof(Vc1ResidualOp) == vc1dsp.RES_DTYPE.itemsize == 16
    for name, _ in Vc1McOp._fields_:
        assert getattr(Vc1McOp, name).offset == vc1dsp.MC_DTYPE.fields[name][1], name
    for name, _ in Vc1McSrc._fields_:
        assert getattr(Vc1McSrc, name).offset == vc1dsp.SRC_DTYPE.fields[name][1], name
    for name, _ in Vc1ResidualOp._fields_:
        assert getattr(Vc1ResidualOp, name).offset == vc1dsp.RES_DTYPE.fields[name][1], name
    assert Vc1McRef.luty.offset == 56 and Vc1McRef.lutuv.offset == 568
    assert C.sizeof(VC1DSPContext) == 95 * 8 and VC1DSPContext.put_vc1_mspel_pixels_tab.offset == 18 * 8
    assert VC1DSPContext.put_no_rnd_vc1_chroma_pixels_tab.offset == 82 * 8 and VC1DSPContext.vc1_unescape_buffer.offset == 94 * 8


# ---------------------------------------------------------------- vc1mc.cu / vc1idct.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emuvc1():
    """libemuvc1.so: vc1mc.cu and vc1idct.cu with their host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The
    kernels with __syncwarp run an OS thread per CUDA thread of a block and __syncwarp becomes the warp's barrier; the residual kernel
    has no collective and runs thread after thread."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vc1mc.cu", "vc1idct.cu", "tx_pfa.cu"):                  # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vc1mc.cu":
            assert t.count("extern __shared__ uint32_t vc1_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { vc1_mc_kernel(") == 1
            t = t.replace("extern __shared__ uint32_t vc1_smem[];", "uint32_t *vc1_smem = (uint32_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { vc1_mc_kernel(", "emu_cfg_launch(2, [&] { vc1_mc_kernel(")
        if f == "vc1idct.cu":
            assert t.count("emu_cfg_launch(0, [&] { vc1_idct_member_kernel(") == 1
            t = t.replace("emu_cfg_launch(0, [&] { vc1_idct_member_kernel(", "emu_cfg_launch(2, [&] { vc1_idct_member_kernel(")
        t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, "vc1_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuvc1.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_vc1_dsp_init.argtypes = [C.c_void_p]
    L.b200_vc1_mc_frame_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int64, C.c_void_p]
    L.b200_vc1_residual_frame_device.argtypes = [C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                                 C.c_void_p]
    L.emu_launch_count.restype = C.c_uint64
    return L


def emu_mc(L, mbw, mbh, H, V, refs, ops, dst):
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    arr = v1.ref_array([r.desc() for r in refs])
    assert L.b200_vc1_mc_frame_device(None, len(refs), C.cast(arr, C.c_void_p), planes, d[0].strides[0], d[1].strides[0], mbw, mbh, H, V, len(ops),
                                      ops.ctypes.data) == 0
    return d


def emu_residual(L, mbw, mbh, ops, coef, dst):
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    assert L.b200_vc1_residual_frame_device(None, planes, d[0].strides[0], d[1].strides[0], mbw, mbh, coef.ctypes.data, len(ops), ops.ctypes.data) == 0
    return d


@pytest.mark.parametrize("name", [c[0] for c in v1.FIXTURE_CASES])
def test_emu_fixture_frames(emuvc1, name):
    """the fixture pictures through both entries: equal to the checker after each, the sentinels outside the MB grid unchanged, and the
    reference's hash at the end"""
    mbw, mbh, H, V, refs, ops, dst, rops, coef = v1.fixture_case(name)
    got = emu_mc(emuvc1, mbw, mbh, H, V, refs, ops, dst)
    exp = v1.orc_mc_frame(mbw, mbh, H, V, refs, ops, dst)
    assert same(got, exp)
    for p, s in zip(got, (16, 8, 8)):
        assert (p[mbh * s:] == v1.SENTINEL).all() and (p[:, mbw * s:] == v1.SENTINEL).all()
    got = emu_residual(emuvc1, mbw, mbh, rops, coef, got)
    assert same(got, v1.orc_residual_frame(mbw, mbh, rops, coef, exp))
    assert v1.digest(got) == v1.fixture_hashes()[name]


@pytest.mark.parametrize("kind", ("decoder", "dense", "extreme"))
def test_emu_residual_vs_checker(emuvc1, kind):
    rng = np.random.default_rng(40 + len(kind))
    rops, coef = v1.residual_case(41 + len(kind), 7, 5, kind)
    dst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v1.dst_planes(7, 5)]
    assert same(emu_residual(emuvc1, 7, 5, rops, coef, dst), v1.orc_residual_frame(7, 5, rops, coef, dst))


def test_emu_invalid_ops_write_nothing(emuvc1):
    """undefined kinds, phases above 3, a reference index >= nrefs, AVG on a 4MV op, destinations not a multiple of 8 or outside the
    grid; residual ops with an undefined plane or ttblk, an unaligned or negative coef_off or a block outside the grid: nothing
    written, while the valid ops of the same call are"""
    refs, ops, dst, H, V = v1.mc_case(51, 4, 3)
    bad = ops[:10].copy()
    bad["kind"][0] = 3
    bad["src"]["mx"][1, 0] = 4
    bad["src"]["uvmy"][2, 0] = 7
    bad["src"]["ref"][3, 0] = 1
    bad["kind"][4], bad["flags"][4] = v1.MC_LUMA8, bad["flags"][4] | v1.AVG
    bad["dst_x"][5] += 4
    bad["dst_y"][6] = -8
    bad["dst_x"][7], bad["kind"][7] = 64, v1.MC_1MV
    bad["dst_y"][8], bad["kind"][8] = 24, v1.MC_CHROMA8
    bad["dst_y"][9], bad["kind"][9] = 48, v1.MC_LUMA8
    assert same(emu_mc(emuvc1, 4, 3, H, V, refs, bad, dst), dst) and same(v1.orc_mc_frame(4, 3, H, V, refs, bad, dst), dst)
    mixed = np.concatenate([bad, ops[10:]])
    got = emu_mc(emuvc1, 4, 3, H, V, refs, mixed, dst)
    assert same(got, v1.orc_mc_frame(4, 3, H, V, refs, mixed, dst)) and not np.array_equal(got[0], dst[0])
    rops, coef = v1.residual_case(52, 4, 3, "dense", skip=0.0)
    rbad = rops[:6].copy()
    rbad["plane"][0], rbad["ttblk"][1], rbad["coef_off"][2], rbad["coef_off"][3], rbad["x"][4], rbad["y"][5] = 3, 4, 4, -64, 60, 48
    rng = np.random.default_rng(53)
    rdst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v1.dst_planes(4, 3)]
    assert same(emu_residual(emuvc1, 4, 3, rbad, coef, rdst), rdst) and same(v1.orc_residual_frame(4, 3, rbad, coef, rdst), rdst)


def test_emu_every_table_entry(emuvc1):
    """every member through host pointers against the checker: all mspel and chroma entries, all transforms on extreme blocks (dest and
    block), and chroma arguments outside the domain writing nothing"""
    from ffmpeg_b200._lib import VC1DSPContext
    from test_vc1_dsp_gpu import check_members
    ctx = VC1DSPContext()
    assert emuvc1.b200_vc1_dsp_init(C.byref(ctx)) == 0
    check_members(ctx, 61)


def test_emu_member_pattern(emuvc1):
    """the transforms and both MC tables filled, chroma [2] and every other member NULL; one function per table position"""
    from ffmpeg_b200._lib import VC1DSPContext
    ctx = VC1DSPContext()
    assert emuvc1.b200_vc1_dsp_init(C.byref(ctx)) == 0
    w = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
    filled = list(range(8)) + list(range(18, 82)) + [82, 83, 85, 86]
    assert (w[filled] != 0).all() and (np.delete(w, filled) == 0).all()
    assert len(set(w[filled].tolist())) == len(filled)
    if v1.have_ref():
        ref = (C.c_void_p * 95)()
        v1.ref().ffref_vc1_pointers(ref)
        words = [x or 0 for x in ref]
        assert all(words[k] for k in filled) and len({words[k] for k in filled}) == len(filled)


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_frame_refusals(prodlib, emuvc1):
    """every B200_EINVAL / B200_ENOSYS case of both entries launches nothing (the buffers stay zero, the stand-in runtime's launch count
    does not move)"""
    from ffmpeg_b200._lib import Vc1McRef
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data
    ops = np.zeros(1, v1.MC_DTYPE)
    rops = np.zeros(1, v1.RES_DTYPE)
    before = emuvc1.emu_launch_count()
    assert prodlib.b200_vc1_dsp_init(None) == EINVAL and emuvc1.b200_vc1_dsp_init(None) == EINVAL
    for L in (prodlib, emuvc1):
        def mc(nrefs=1, n=1, ops=ops.ctypes.data, refs=True, planes=(p + 1024, p + 4096, p + 8192), ls_y=64, ls_uv=32, mbw=2, mbh=2, H=32, V=32,
               ref_planes=(p + 16384, p + 20480, p + 24576), interlaced=(0, 0)):
            arr = (Vc1McRef * 2)(*[Vc1McRef(*ref_planes, 64, 32, 0, 0, interlaced[k], 0) for k in range(2)])
            dp = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vc1_mc_frame_device(None, nrefs, C.cast(arr, C.c_void_p) if refs else None, dp, ls_y, ls_uv, mbw, mbh, H, V, n, ops)
        assert mc(n=0) == 0 and mc(n=0, ops=None, refs=False, planes=None) == 0
        assert mc(n=-1) == EINVAL and mc(nrefs=0) == EINVAL and mc(nrefs=3) == EINVAL
        assert mc(mbw=0) == EINVAL and mc(mbh=2048) == EINVAL and mc(H=0) == EINVAL and mc(V=32768) == EINVAL
        assert mc(ops=None) == EINVAL and mc(refs=False) == EINVAL and mc(planes=None) == EINVAL and mc(ops=ops.ctypes.data + 2) == EINVAL
        assert mc(ls_y=66) == EINVAL and mc(ls_uv=34) == EINVAL
        for k in range(3):
            pl = [p + 1024, p + 4096, p + 8192]
            pl[k] = 0
            assert mc(planes=tuple(pl)) == EINVAL, k
            pl[k] = [p + 1025, p + 4098, p + 8195][k]
            assert mc(planes=tuple(pl)) == EINVAL, k
            rp = [p + 16384, p + 20480, p + 24576]
            rp[k] = 0
            assert mc(ref_planes=tuple(rp)) == EINVAL, k
        assert mc(interlaced=(1, 0)) == ENOSYS and mc(nrefs=2, interlaced=(0, 1)) == ENOSYS

        def res(n=1, ops=rops.ctypes.data, coef=p + 32768, planes=(p + 1024, p + 4096, p + 8192), ls_y=64, ls_uv=32, mbw=2, mbh=2):
            dp = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vc1_residual_frame_device(None, dp, ls_y, ls_uv, mbw, mbh, coef, n, ops)
        assert res(n=0) == 0 and res(n=0, ops=None, coef=None, planes=None) == 0
        assert res(n=-1) == EINVAL and res(mbw=0) == EINVAL and res(mbh=-1) == EINVAL and res(mbw=2048) == EINVAL
        assert res(ops=None) == EINVAL and res(coef=None) == EINVAL and res(planes=None) == EINVAL
        assert res(ops=rops.ctypes.data + 4) == EINVAL and res(coef=p + 32776) == EINVAL
        assert res(planes=(p + 1026, p + 4096, p + 8192)) == EINVAL and res(planes=(p + 1024, 0, p + 8192)) == EINVAL
        assert res(ls_y=62) == EINVAL and res(ls_uv=30) == EINVAL
    assert not b.any()
    assert emuvc1.emu_launch_count() == before
