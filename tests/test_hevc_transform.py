"""CPU tier for the HEVC residual (HEVCDSPContext's transform members and b200_hevc_transform_add_batch_device,
ffmpeg_b200/csrc/hevcidct.cu): the checker (oracle/hevcidct_oracle.c) against the compiled reference (oracle/_ref/libffref_hevcidct.so)
member by member and on the decoder's batch sequence, the fixture hashes, the ctypes mirror, and hevcidct.cu itself, host code included,
on the stand-in CUDA runtime of tests/cuda_emu (the batch entry, sentinels, every member of every depth, invalid ops and the refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import hevcidctlib as hi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", hi.DEPTHS)
@pytest.mark.parametrize("cls", hi.CLASSES)
def test_checker_members_match_reference(depth, cls):
    """idct (col_limit from the decoder, small, negative and oversized), idct_dc, transform_4x4_luma, dequant and transform_rdpcm at
    every size, on parser-shaped, dense, extreme-valued blocks"""
    seed = 100 + 13 * depth + hi.CLASSES.index(cls)
    ours = hi.run_members(cl.oracle(), "orc_hevc_tx", seed, depth, cls)
    with hi.RefCheck() as rc:
        assert rc.same(ours, lambda: hi.run_members(hi.ref(), "ffref_hevc_tx", seed, depth, cls))


@pytest.mark.parametrize("depth", hi.DEPTHS)
def test_checker_add_residual_matches_reference(depth):
    calls = list(hi.residual_calls(40 + depth, depth))
    ours = [hi.run_add(cl.oracle(), "orc_hevc_add_residual", depth, c) for c in calls]
    with hi.RefCheck() as rc:
        assert rc.same(ours, lambda: [hi.run_add(hi.ref(), "ffref_hevc_add_residual", depth, c) for c in calls])


@pytest.mark.parametrize("depth", hi.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_checker_batch_matches_decoder_sequence(depth, chroma):
    """the checker's batch against the reference driver's member calls (cabac.c:1550-1592, then add_residual), per input class"""
    for cls in hi.CLASSES:
        case = hi.batch_case(300 + depth + chroma + hi.CLASSES.index(cls), 200, depth, bool(chroma), cls=cls)
        ours = hi.orc_batch(depth, *case)
        assert not np.array_equal(ours, case[1])
        with hi.RefCheck() as rc:
            assert rc.same(ours, lambda: hi.ref_batch(depth, *case))


def test_checker_reproduces_fixture():
    hs = hi.fixture_hashes()
    assert len(hs) == len(hi.DEPTHS) * 2
    for (depth, chroma), h in hs.items():
        assert hi.digest(hi.orc_batch(depth, *hi.fixture_case(depth, int(chroma)))) == h, (depth, chroma)


def test_ctypes_mirror():
    from ffmpeg_b200._lib import HevcTuOp
    from ffmpeg_b200 import hevcdsp
    assert C.sizeof(HevcTuOp) == hevcdsp.TU_DTYPE.itemsize == 32
    for name, _ in HevcTuOp._fields_:
        assert getattr(HevcTuOp, name).offset == hevcdsp.TU_DTYPE.fields[name][1], name


# ---------------------------------------------------------------- hevcidct.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emuidct():
    """libemuhevcidct.so: hevcidct.cu and hevcmc.cu with their host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.
    The kernels use shared memory and __syncthreads, so they run an OS thread per CUDA thread of a block (emu.h's block launch)."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("hevcidct.cu", "hevcmc.cu", "tx_pfa.cu"):           # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "hevcidct.cu":
            assert t.count("extern __shared__ int4 hevc_tu_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { hevc_tu_kernel<") == 2
            t = t.replace("extern __shared__ int4 hevc_tu_smem[];", "int4 *hevc_tu_smem = (int4 *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_tu_kernel<", "emu_cfg_launch(2, [&] { hevc_tu_kernel<")
        if f == "hevcmc.cu":
            t = t.replace("extern __shared__ int16_t hevc_smem[];", "int16_t *hevc_smem = (int16_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_mc_kernel<", "emu_cfg_launch(2, [&] { hevc_mc_kernel<")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, "idct_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuhevcidct.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_hevc_dsp_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_hevc_dsp_init_transform.argtypes = [C.c_void_p, C.c_int]
    L.b200_hevc_transform_add_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t]
    L.emu_launch_count.restype = C.c_uint64
    L.b200_last_error.restype = C.c_char_p
    return L


def emu_batch(L, depth, coef, dst, ops):
    d, c = dst.copy(), coef.copy()
    assert L.b200_hevc_transform_add_batch_device(None, depth, len(ops), ops.ctypes.data, c.ctypes.data, d.ctypes.data, d.strides[0]) == 0
    assert np.array_equal(c, coef)
    return d


@pytest.mark.parametrize("depth", hi.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_emu_batch_vs_checker_and_fixture(emuidct, depth, chroma):
    """the fixture batch through the library's entry: equal to the checker over the whole destination (the sentinels around and
    between the blocks unchanged, coef unchanged) and to the reference's hash"""
    case = hi.fixture_case(depth, chroma)
    got = emu_batch(emuidct, depth, *case)
    assert np.array_equal(got, hi.orc_batch(depth, *case))
    assert hi.digest(got) == hi.fixture_hashes()[(depth, bool(chroma))]
    outside = np.ones(got.shape, bool)
    for o in case[2]:
        y, x, n = o["dst_off"] // got.strides[0], o["dst_off"] % got.strides[0] // got.itemsize, 1 << o["log2_size"]
        outside[y:y + n, x:x + n] = False
    assert (got[outside] == case[1][0, 0]).all()


def test_emu_invalid_ops_write_nothing(emuidct):
    """log2_size outside 2..5, undefined kinds, DST4 above 4x4, coef_off not a multiple of 8, dst_off not a multiple of 4 samples"""
    for depth in (8, 10):
        coef, dst, ops = hi.batch_case(51, 16, depth)
        bad = ops.copy()
        bad["log2_size"][0], bad["log2_size"][1], bad["log2_size"][2] = 1, 6, 255
        bad["kind"][3], bad["kind"][4] = 5, 255
        bad["kind"][5], bad["log2_size"][5] = 2, 3
        bad["coef_off"][6] += 4
        bad["dst_off"][7] += dst.itemsize * 2
        bad["coef_off"][8] += 1
        assert np.array_equal(emu_batch(emuidct, depth, coef, dst, bad[:9]), dst)
        assert np.array_equal(hi.orc_batch(depth, coef, dst, bad[:9]), dst)


def test_emu_every_member(emuidct):
    """all 15 member pointers at every depth, called through the context with host pointers, against the checker"""
    from ffmpeg_b200._lib import HEVCDSPContext
    for depth in hi.DEPTHS:
        ctx = HEVCDSPContext()
        assert emuidct.b200_hevc_dsp_init(C.byref(ctx), depth) == 0
        assert emuidct.b200_hevc_dsp_init_transform(C.byref(ctx), depth) == 0
        for cls in ("decoder", "odd_limit", "extreme"):
            for call in hi.member_calls(80 + depth, depth, cls):
                assert np.array_equal(hi.ctx_tx(ctx, call), hi.run_tx(cl.oracle(), "orc_hevc_tx", depth, call)), (depth, call[0], call[1], call[3])
        for call in hi.residual_calls(90 + depth, depth):
            assert np.array_equal(hi.ctx_add(ctx, call), hi.run_add(cl.oracle(), "orc_hevc_add_residual", depth, call))


def test_emu_members_refuse_bad_log2(emuidct):
    """dequant / transform_rdpcm with log2_size outside 2..5 write nothing, launch nothing and say why"""
    from ffmpeg_b200._lib import HEVCDSPContext
    from ffmpeg_b200 import hevcdsp as hd
    ctx = HEVCDSPContext()
    assert emuidct.b200_hevc_dsp_init_transform(C.byref(ctx), 10) == 0
    c = np.arange(64 * 64, dtype=np.int16)
    before = emuidct.emu_launch_count()
    for log2 in (0, 1, 6, -1):
        hd.DEQUANT(ctx.dequant)(c.ctypes.data, log2)
        hd.TRANSFORM_RDPCM(ctx.transform_rdpcm)(c.ctypes.data, log2, 1)
    assert np.array_equal(c, np.arange(64 * 64, dtype=np.int16)) and emuidct.emu_launch_count() == before
    assert b"log2_size" in emuidct.b200_last_error()


def test_emu_init_sets_exactly_the_residual_members(emuidct):
    """after b200_hevc_dsp_init: the MC tables are unchanged, the 15 residual function pointers are set, every other member stays NULL"""
    from ffmpeg_b200._lib import HEVCDSPContext
    ctx = HEVCDSPContext()
    assert emuidct.b200_hevc_dsp_init(C.byref(ctx), 12) == 0
    before = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64).copy()
    assert emuidct.b200_hevc_dsp_init_transform(C.byref(ctx), 12) == 0
    words = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
    res = np.zeros(len(words), bool)
    res[1:1 + 4 + 3 + 4 + 4] = True                    # add_residual[4], dequant, transform_rdpcm, transform_4x4_luma, idct[4], idct_dc[4]
    assert res.sum() == 15
    assert (words[res] != 0).all() and (before[res] == 0).all()
    assert np.array_equal(words[~res], before[~res])
    blank = HEVCDSPContext()
    assert emuidct.b200_hevc_dsp_init_transform(C.byref(blank), 8) == 0
    w2 = np.frombuffer(C.string_at(C.addressof(blank), C.sizeof(blank)), np.uint64)
    assert (w2[res] != 0).all() and (w2[~res] == 0).all()


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emuidct):
    from ffmpeg_b200._lib import HEVCDSPContext
    for L in (prodlib, emuidct):
        ctx = HEVCDSPContext()
        for depth in (0, 7, 11, 13, 14, 16):
            assert L.b200_hevc_dsp_init_transform(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_hevc_dsp_init_transform(None, 8) == EINVAL


def test_batch_refusals(prodlib, emuidct):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    b = np.zeros(8192 + 64, np.uint8)
    base = (b.ctypes.data + 63) & ~63
    ops = np.zeros(2, hi.TU_DTYPE)
    ops["log2_size"] = 2
    o = (ops.ctypes.data + 15) & ~15 if ops.ctypes.data & 15 else ops.ctypes.data
    before = emuidct.emu_launch_count()
    for L in (prodlib, emuidct):
        def call(depth=8, n=1, ops=o, coef=base + 4096, dst=base, ds=64):
            return L.b200_hevc_transform_add_batch_device(None, depth, n, ops, coef, dst, ds)
        assert call(n=0) == 0 and call(n=0, ops=None, coef=None, dst=None) == 0
        assert call(n=-1) == EINVAL
        for depth in (0, 7, 11, 13, 14, 16):
            assert call(depth=depth) == EINVAL, depth
        assert call(ds=62) == EINVAL and call(ds=2) == EINVAL and call(depth=10, ds=4) == EINVAL and call(depth=10, ds=68) == EINVAL
        for k in ("ops", "coef", "dst"):
            assert call(**{k: None}) == EINVAL, k
        assert call(ops=o + 8) == EINVAL and call(coef=base + 4096 + 8) == EINVAL and call(dst=base + 2) == EINVAL
        assert call(depth=10, dst=base + 4) == EINVAL
    assert not b.any()
    assert emuidct.emu_launch_count() == before
