"""CPU tier for HEVC intra prediction (HEVCPredContext and b200_hevc_intra_pred_batch_device, ffmpeg_b200/csrc/hevcpred.cu): hevcpred.cu
itself, host code included, on the stand-in CUDA runtime of tests/cuda_emu, against the reference's own intra_pred (live where
oracle/_ref/libffref_hevcpred.so is built, stored digests elsewhere): whole planes through the level wavefront for luma and 4:2:0 /
4:2:2 / 4:4:4 chroma with constrained intra prediction on and off, guard samples unchanged; every member at every depth; the
strong-smoothing decision at its threshold; the fixture hashes; which members init sets; the refusals, with no launch.  The checker
(oracle/hevcpred_oracle.c) is pinned to the reference on the same members and planes, and the library is compared with it too."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hevcpredlib as hl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


@pytest.fixture(scope="module")
def emupred():
    """libemuhevcpred.so: hevcpred.cu with its host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The kernels use
    shared memory and __syncthreads, so they run one OS thread per CUDA thread of a block (emu.h's block launch)."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("hevcpred.cu", "tx_pfa.cu"):                          # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "hevcpred.cu":
            assert t.count("extern __shared__ int ipred_smem[];") == 2
            assert t.count("emu_cfg_launch(0, [&] { hevc_intra_kernel<") == 2 and t.count("emu_cfg_launch(0, [&] { hevc_pred_member_kernel<") == 1
            t = t.replace("extern __shared__ int ipred_smem[];", "int *ipred_smem = (int *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_", "emu_cfg_launch(2, [&] { hevc_")
        assert "<<<" not in t
        p = os.path.join(gen, "ipred_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuhevcpred.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_hevc_pred_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_hevc_intra_pred_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int]
    L.emu_launch_count.restype = C.c_uint64
    L.b200_last_error.restype = C.c_char_p
    return L


def emu_plane(L, p):
    """the component through the level wavefront: one library call per level, then the residual added on the host"""
    m = None if p.map is None else np.ascontiguousarray(p.map)

    def call(buf, ops):
        assert L.b200_hevc_intra_pred_batch_device(None, p.depth, hl._ptr(buf), buf.strides[0], p.W, p.H, p.hs, p.vs, len(ops), ops.ctypes.data,
                                                   None if m is None else m.ctypes.data, 0 if m is None else m.strides[0], p.log2_min_pu) == 0
    return hl.run_levels(p, call)[0]


PICTURES = [  # (W, H, log2_ctb, kwargs): luma sizes not multiples of the CTB
    (200, 136, 4, dict(nslices=3)),
    (232, 120, 5, dict(tiles=(2, 2), nslices=2)),
    (200, 136, 6, dict(nslices=2, smoothing=False)),
    (136, 72, 5, dict(nslices=1, strong=False, tiles=(2, 1))),
]


@pytest.mark.parametrize("cip", (False, True), ids=("nocip", "cip"))
@pytest.mark.parametrize("name", ("luma", "420", "422", "444"))
def test_emu_plane_is_the_decoder(emupred, name, cip):
    """the library's level wavefront against the reference's intra_pred TU by TU, at 8 and 10 bit, CTB 16 / 32 / 64, slices and tiles,
    smoothing and strong smoothing on and off; the guard samples around the plane unchanged"""
    cfmt, comp = hl.FIXTURE_CFMT[name]
    for depth in (8, 10):
        for k, (W, H, l2, kw) in enumerate(PICTURES):
            p = hl.picture_case(100 * depth + 10 * k + 2 * cfmt + int(cip), depth, W, H, l2, cfmt, comp, cip=cip, **kw)
            got = emu_plane(emupred, p)
            guard = got.copy()
            guard[hl.MARGIN:hl.MARGIN + p.ph, hl.MARGIN:hl.MARGIN + p.pw] = hl.sentinel(depth)
            assert (guard == hl.sentinel(depth)).all()
            assert np.array_equal(got, hl.orc_plane(p)), (depth, k)
            with hl.RefCheck() as rc:
                assert rc.same(got, lambda: hl.ref_plane(p)), (depth, k)


@pytest.mark.parametrize("cip", (False, True), ids=("nocip", "cip"))
@pytest.mark.parametrize("name", ("luma", "420", "422", "444"))
def test_checker_plane_is_the_decoder(name, cip):
    """the checker's level wavefront against the reference's intra_pred TU by TU, at every depth, on other seeds than the library's"""
    cfmt, comp = hl.FIXTURE_CFMT[name]
    for depth in hl.DEPTHS:
        for k, (W, H, l2, kw) in enumerate(PICTURES):
            p = hl.picture_case(5000 + 100 * depth + 10 * k + 2 * cfmt + int(cip), depth, W, H, l2, cfmt, comp, cip=cip, **kw)
            ours = hl.orc_plane(p)
            with hl.RefCheck() as rc:
                assert rc.same(ours, lambda: hl.ref_plane(p)), (depth, k)


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_checker_members_match_reference(depth):
    """the checker's planar / DC / angular (every size x mode x luma / chroma) and both filters against the reference"""
    cases = list(hl.member_cases(900 + depth, depth))
    ours = [hl.orc_member(depth, c) for c in cases]
    with hl.RefCheck() as rc:
        assert rc.same(ours, lambda: [hl.ref_member(depth, c) for c in cases])
    fcases = list(hl.filter_cases(950 + depth, depth))
    ours = [a for c in fcases for a in hl.orc_filters(depth, c)]
    with hl.RefCheck() as rc:
        assert rc.same(ours, lambda: [a for c in fcases for a in hl.ref_filters(depth, c)])


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_emu_strong_threshold(emupred, depth):
    """32x32 luma blocks whose strong-smoothing second differences lie at t - 1 and t (t = 1 << (depth - 5)) on either side, top and
    left: the library equals the checker and the reference, and the cases take both outcomes of the decision"""
    p = hl.strong_case(40 + depth, depth)
    got = emu_plane(emupred, p)
    assert np.array_equal(got, hl.orc_plane(p))
    with hl.RefCheck() as rc:
        assert rc.same(got, lambda: hl.ref_plane(p))
    q = hl.strong_case(40 + depth, depth)
    q.ops["flags"] &= np.uint16(0xFFFF & ~hl.INTRA_STRONG)
    plain = hl.orc_plane(q)
    same = [np.array_equal(hl.inner(got, p)[y:y + 32, x:x + 32], hl.inner(plain, q)[y:y + 32, x:x + 32]) for x, y, *_ in p.tus]
    assert same == [False, True, True, False, True, True, True, False], same


def test_fixture_hashes(emupred):
    """the fixture planes (every depth x luma / 4:2:0 / 4:2:2 / 4:4:4 x CIP off / on) through the library equal the stored hashes of the
    reference's planes"""
    hs = hl.fixture_hashes()
    assert len(hs) == len(hl.DEPTHS) * 8
    for depth in hl.DEPTHS:
        for name in hl.FIXTURE_CFMT:
            for cip in (False, True):
                assert hl.digest(emu_plane(emupred, hl.fixture_case(depth, name, cip))) == hs[(depth, hl.fixture_key(name, cip))]


def test_fixture_is_the_reference_result():
    if not hl.have_ref():
        pytest.skip("the reference is not built here; test_fixture_hashes checks the stored hashes")
    hs = hl.fixture_hashes()
    for depth in hl.DEPTHS:
        for name in hl.FIXTURE_CFMT:
            for cip in (False, True):
                assert hl.digest(hl.ref_plane(hl.fixture_case(depth, name, cip))) == hs[(depth, hl.fixture_key(name, cip))]


def _ctx(L, depth):
    from ffmpeg_b200._lib import HEVCPredContext
    ctx = HEVCPredContext()
    assert L.b200_hevc_pred_init(C.byref(ctx), depth) == 0
    return ctx


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_emu_every_member(emupred, depth):
    """planar / DC / angular at every size x every mode x luma / chroma, and both filters, against the reference (guards included)"""
    ctx = _ctx(emupred, depth)
    cases = list(hl.member_cases(700 + depth, depth))
    ours = [hl.ctx_member(ctx, depth, c) for c in cases]
    assert all(np.array_equal(a, hl.orc_member(depth, c)) for a, c in zip(ours, cases))
    with hl.RefCheck() as rc:
        assert rc.same(ours, lambda: [hl.ref_member(depth, c) for c in cases])
    fcases = list(hl.filter_cases(800 + depth, depth))
    ours = [a for k, c in enumerate(fcases) for a in hl.ctx_filters(ctx, depth, c, k % 3)]
    with hl.RefCheck() as rc:
        assert rc.same(ours, lambda: [a for k, c in enumerate(fcases) for a in hl.ref_filters(depth, c, k % 3)])


def test_emu_filters_launch_nothing_and_domain(emupred):
    from ffmpeg_b200 import hevcdsp as hd
    ctx = _ctx(emupred, 10)
    before = emupred.emu_launch_count()
    for c in hl.filter_cases(5, 10):
        hl.ctx_filters(ctx, 10, c)
    assert emupred.emu_launch_count() == before
    t = np.arange(160, dtype=np.uint16)
    d = np.full((40, 40), 7, np.uint16)
    for mode in (-1, 0, 1, 35, 255):
        hd.PRED_ANGULAR(ctx.pred_angular[1])(d.ctypes.data, t.ctypes.data + 2, t.ctypes.data + 2, 40, 0, mode)
    for log2 in (1, 6, -1):
        hd.PRED_DC(ctx.pred_dc)(d.ctypes.data, t.ctypes.data + 2, t.ctypes.data + 2, 40, log2, 0)
    assert (d == 7).all() and emupred.emu_launch_count() == before
    assert b"log2_size" in emupred.b200_last_error()


def test_emu_init_sets_exactly_the_members(emupred):
    """every member but intra_pred[] is set; intra_pred[] is NULL; the three 3-tap pointers are one function"""
    from ffmpeg_b200._lib import HEVCPredContext
    ctx = HEVCPredContext()
    C.memset(C.addressof(ctx), 0x11, C.sizeof(ctx))
    assert emupred.b200_hevc_pred_init(C.byref(ctx), 12) == 0
    assert not any(ctx.intra_pred)
    assert all(ctx.pred_planar) and ctx.pred_dc and all(ctx.pred_angular) and ctx.ref_filter_strong
    assert len(set(ctx.ref_filter_3tap)) == 1 and ctx.ref_filter_3tap[0]
    assert len(set(ctx.pred_planar)) == 4 and len(set(ctx.pred_angular)) == 4


def test_ctypes_mirrors():
    from ffmpeg_b200._lib import HevcIntraOp, HEVCPredContext
    from ffmpeg_b200 import hevcdsp
    assert C.sizeof(HevcIntraOp) == hevcdsp.INTRA_DTYPE.itemsize == 16
    for name, _ in HevcIntraOp._fields_:
        assert getattr(HevcIntraOp, name).offset == hevcdsp.INTRA_DTYPE.fields[name][1], name
    assert C.sizeof(HEVCPredContext) == 17 * 8
    if hl.have_ref():
        assert bytes((C.c_char * 19).in_dll(hl.ref(), "ffref_hevcpred_layout_check")) == b"B200HEVCPredContext"


def test_out_of_range_ops_change_nothing(emupred):
    """ops with a bad size or mode, or whose block or flagged neighbours fall outside the plane, write nothing"""
    p = hl.picture_case(3, 8, 64, 64, 5, 0, 0)
    buf = hl.framed(p.plane, 8)
    bad = np.zeros(9, hl.INTRA_DTYPE)
    bad[:] = [(0, 0, 1, 0, 0, (0,) * 4), (0, 0, 6, 0, 0, (0,) * 4), (8, 8, 2, 35, 0, (0,) * 4), (-4, 0, 2, 0, 0, (0,) * 4),
              (0, -4, 2, 0, 0, (0,) * 4), (60, 0, 3, 0, 0, (0,) * 4), (0, 60, 3, 0, 0, (0,) * 4),
              (0, 8, 2, 0, hl.INTRA_CAND_L, (0,) * 4), (8, 0, 2, 0, hl.INTRA_CAND_U, (0,) * 4)]
    before = buf.copy()
    assert emupred.b200_hevc_intra_pred_batch_device(None, 8, hl._ptr(buf), buf.strides[0], 64, 64, 0, 0, len(bad), bad.ctypes.data, None, 0, 2) == 0
    assert np.array_equal(buf, before)


@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emupred):
    from ffmpeg_b200._lib import HEVCPredContext
    for L in (prodlib, emupred):
        ctx = HEVCPredContext()
        for depth in (0, 7, 11, 13, 14, 16):
            assert L.b200_hevc_pred_init(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_hevc_pred_init(None, 8) == EINVAL
        assert not any(bytes(ctx))


def test_batch_refusals(prodlib, emupred):
    """every B200_EINVAL case launches nothing and writes nothing; nops == 0 returns 0"""
    mem = np.zeros(64 * 128 + 64, np.uint8)
    pix = (mem.ctypes.data + 63) & ~63
    o = np.zeros(4 + 1, hl.INTRA_DTYPE)
    ops = (o.ctypes.data + 15) & ~15
    m = np.ones(4096, np.uint8)
    before = emupred.emu_launch_count()
    for L in (prodlib, emupred):
        def call(depth=8, px=pix, st=128, W=64, H=64, hs=0, vs=0, n=4, op=ops, mp=None, ms=0, pu=2):
            return L.b200_hevc_intra_pred_batch_device(None, depth, px, st, W, H, hs, vs, n, op, mp, ms, pu)
        assert call(px=None) == EINVAL and call(op=None) == EINVAL and call(n=-1) == EINVAL
        for depth in (0, 7, 11, 13, 16):
            assert call(depth=depth) == EINVAL, depth
        for W, H in ((0, 8), (8, 0), (-8, 8)):
            assert call(W=W, H=H) == EINVAL
        for hs, vs in ((2, 0), (0, 2), (-1, 0)):
            assert call(hs=hs, vs=vs) == EINVAL
        assert call(st=63) == EINVAL and call(st=-128) == EINVAL and call(depth=10, st=127) == EINVAL
        assert call(depth=10, px=pix + 1, W=32) == EINVAL and call(op=ops + 8) == EINVAL
        assert call(mp=m.ctypes.data, ms=15) == EINVAL and call(mp=m.ctypes.data, ms=16, pu=1) == EINVAL
        assert call(mp=m.ctypes.data, ms=16, pu=7) == EINVAL
        assert call(n=0) == 0 and call(n=0, px=None, op=None) == 0
    assert not mem.any() and emupred.emu_launch_count() == before
