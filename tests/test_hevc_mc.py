"""CPU tier for HEVC motion compensation (HEVCDSPContext's put_hevc_* tables, ffmpeg_b200/csrc/hevcmc.cu): the checker
(oracle/hevcmc_oracle.c) against the compiled reference (oracle/_ref/libffref_hevcdsp.so) member by member and on the decoder's batch
sequence, the fixture hashes, the layout marker, and hevcmc.cu itself, host code included, on the stand-in CUDA runtime of tests/cuda_emu
(the batch entry, sentinels, every table entry of every depth, and the refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import hevcmclib as hm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", hm.DEPTHS)
@pytest.mark.parametrize("epel", (0, 1), ids=("qpel", "epel"))
@pytest.mark.parametrize("cls", (0, 1, 2, 3), ids=("noise", "zero", "max", "extremes"))
def test_checker_members_match_reference(depth, epel, cls):
    """every (form, [v][h], width) member with every phase pair in turn, src2 over the int16 range, weights and offsets at their ends"""
    seed = 100 + 13 * depth + 3 * epel + cls
    ours = hm.run_members(cl.oracle(), "orc_hevc_mc", seed, depth, epel, cls)
    with hm.RefCheck() as rc:
        assert rc.same(ours, lambda: hm.run_members(hm.ref(), "ffref_hevc_mc", seed, depth, epel, cls))


@pytest.mark.parametrize("depth", hm.DEPTHS)
@pytest.mark.parametrize("epel", (0, 1), ids=("luma", "chroma"))
def test_checker_batch_matches_decoder_sequence(depth, epel):
    """the checker's clamped reads against the reference driver's emulated_edge_mc windows + member calls: blocks at every edge and
    corner, windows wholly outside (positions up to 80 samples beyond the picture), bi ops with one integer and one fractional reference"""
    for cls in (0, 3):
        case = hm.batch_case(300 + depth + epel + cls, 768, depth, epel, cls=cls)
        ours = hm.orc_batch(depth, epel, *case)
        assert not np.array_equal(ours, case[1])
        with hm.RefCheck() as rc:
            assert rc.same(ours, lambda: hm.ref_batch(depth, epel, *case))


def test_context_layout_matches_reference():
    """oracle/ref/ref_hevcdsp.c asserts at compile time that B200HEVCDSPContext has HEVCDSPContext's size, member offsets and
    function-pointer types: the marker proves the unit was compiled"""
    if not hm.have_ref():
        pytest.skip("oracle/_ref/libffref_hevcdsp.so not built")
    marker = C.c_char_p.in_dll(hm.ref(), "ffref_hevcdsp_layout_check")
    assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200HEVCDSPContext matches")


def test_checker_reproduces_fixture():
    hs = hm.fixture_hashes()
    assert len(hs) == len(hm.DEPTHS) * 2
    for (depth, epel), h in hs.items():
        assert hm.digest(hm.orc_batch(depth, int(epel), *hm.fixture_case(depth, int(epel)))) == h, (depth, epel)


def test_ctypes_mirrors():
    from ffmpeg_b200._lib import HEVCDSPContext, HevcMcOp
    from ffmpeg_b200 import hevcdsp
    assert C.sizeof(HevcMcOp) == hevcdsp.OP_DTYPE.itemsize == 64
    for name, _ in HevcMcOp._fields_:
        assert getattr(HevcMcOp, name).offset == hevcdsp.OP_DTYPE.fields[name][1], name
    assert C.sizeof(HEVCDSPContext) == (28 + 10 * 40 + 8) * 8 and HEVCDSPContext.put_hevc_qpel.offset == 28 * 8


# ---------------------------------------------------------------- hevcmc.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emuhevc():
    """libemuhevc.so: hevcmc.cu with its host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The kernel uses
    shared memory, __syncthreads and __syncwarp, so it runs an OS thread per CUDA thread of a block (emu.h's block launch), and
    __syncwarp becomes the warp's barrier."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("hevcmc.cu", "tx_pfa.cu"):                          # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "hevcmc.cu":
            assert t.count("extern __shared__ int16_t hevc_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { hevc_mc_kernel<") == 4
            t = t.replace("extern __shared__ int16_t hevc_smem[];", "int16_t *hevc_smem = (int16_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_mc_kernel<", "emu_cfg_launch(2, [&] { hevc_mc_kernel<")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, "hevc_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuhevc.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_hevc_dsp_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_hevc_mc_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_void_p,
                                            C.c_ssize_t, C.c_int, C.c_int]
    return L


def emu_batch(L, depth, epel, ref, dst, ops):
    d = dst.copy()
    r = L.b200_hevc_mc_batch_device(None, depth, epel, len(ops), ops.ctypes.data, d.ctypes.data, d.strides[0], ref.ctypes.data + ref.strides[0],
                                    ref.strides[1], ref.shape[2], ref.shape[1])
    assert r == 0
    return d


@pytest.mark.parametrize("depth", hm.DEPTHS)
@pytest.mark.parametrize("epel", (0, 1), ids=("luma", "chroma"))
def test_emu_batch_vs_checker_and_fixture(emuhevc, depth, epel):
    """the fixture batch through the library's entry: equal to the checker over the whole destination (the sentinels around and
    between the blocks unchanged) and to the reference's hash"""
    case = hm.fixture_case(depth, epel)
    got = emu_batch(emuhevc, depth, epel, *case)
    exp = hm.orc_batch(depth, epel, *case)
    assert np.array_equal(got, exp)
    assert hm.digest(got) == hm.fixture_hashes()[(depth, bool(epel))]
    sentinel = case[1][0, 0]
    assert (got == sentinel).sum() >= case[1].size - int((case[2]["w"].astype(int) * case[2]["h"]).sum())


def test_emu_invalid_ops_write_nothing(emuhevc):
    """w / h outside 1..64, undefined kinds, phases out of range, denom above 7, odd offsets at 16 bit: nothing written"""
    for depth, epel in ((8, 0), (10, 1)):
        ref, dst, ops = hm.batch_case(51, 16, depth, epel)
        bad = ops.copy()
        P = 8 if epel else 4
        bad["w"][0], bad["h"][1], bad["w"][2], bad["h"][3] = 0, 0, 65, 65
        bad["kind"][4], bad["kind"][5] = 4, 255
        bad["mx"][6, 0], bad["my"][7, 0], bad["kind"][8], bad["mx"][8, 1] = P, P, 2, P
        bad["denom"][9] = 8
        bad["kind"][10], bad["mx"][10, 0] = 0, 255
        if depth > 8:
            bad["dst_off"][11] += 1
            bad["kind"][12], bad["ref_off"][12, 1] = 3, 1
        n = 13 if depth > 8 else 11
        assert np.array_equal(emu_batch(emuhevc, depth, epel, ref, dst, bad[:n]), dst)
        assert np.array_equal(hm.orc_batch(depth, epel, ref, dst, bad[:n]), dst)


def test_emu_every_table_entry(emuhevc):
    """every entry [idx][v][h] of the ten tables at every depth, called once with host pointers, against the checker"""
    from ffmpeg_b200._lib import HEVCDSPContext
    from test_hevc_mc_gpu import run_ctx_member
    for depth in hm.DEPTHS:
        ctx = HEVCDSPContext()
        assert emuhevc.b200_hevc_dsp_init(C.byref(ctx), depth) == 0
        for epel in (0, 1):
            pic, src2, dst0 = hm.member_case(70 + depth + epel, depth, epel, 0)
            for call in hm.member_calls(70 + depth + epel, depth, epel):
                exp = hm.run_member(cl.oracle(), "orc_hevc_mc", depth, epel, call, pic, src2, dst0)
                assert np.array_equal(run_ctx_member(ctx, depth, epel, call, pic, src2, dst0), exp), (depth, epel, call)


def test_emu_member_null_pattern(emuhevc):
    """the six inter-prediction tables filled for both filters, every other member NULL"""
    from ffmpeg_b200._lib import HEVCDSPContext
    ctx = HEVCDSPContext()
    assert emuhevc.b200_hevc_dsp_init(C.byref(ctx), 10) == 0
    words = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
    filled = np.zeros(len(words), bool)
    filled[28:28 + 400] = True
    assert (words[filled] != 0).all() and (words[~filled] == 0).all()


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emuhevc):
    from ffmpeg_b200._lib import HEVCDSPContext
    for L in (prodlib, emuhevc):
        ctx = HEVCDSPContext()
        for depth in (0, 7, 11, 13, 14, 16):
            assert L.b200_hevc_dsp_init(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_hevc_dsp_init(None, 8) == EINVAL


def test_batch_refusals(prodlib, emuhevc):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    b = np.zeros(4096, np.uint8)
    p = b.ctypes.data
    ops = np.zeros(1, hm.OP_DTYPE)
    ops["w"] = ops["h"] = 4
    o = ops.ctypes.data
    emuhevc.emu_launch_count.restype = C.c_uint64
    before = emuhevc.emu_launch_count()
    for L in (prodlib, emuhevc):
        def call(depth=8, epel=0, n=1, ops=o, dst=p + 64, ds=64, ref=p + 2048, rs=64, w=16, h=16):
            return L.b200_hevc_mc_batch_device(None, depth, epel, n, ops, dst, ds, ref, rs, w, h)
        assert call(n=0) == 0 and call(n=0, ops=None, dst=None, ref=None) == 0
        assert call(n=-1) == EINVAL
        for depth in (0, 7, 11, 13, 14, 16):
            assert call(depth=depth) == EINVAL, depth
        for epel in (-1, 2):
            assert call(epel=epel) == EINVAL
        assert call(w=0) == EINVAL and call(h=0) == EINVAL and call(w=-5) == EINVAL
        assert call(depth=10, ds=63) == EINVAL and call(depth=10, rs=65) == EINVAL
        for k in ("ops", "dst", "ref"):
            assert call(**{k: None}) == EINVAL, k
        assert call(depth=10, dst=p + 65) == EINVAL and call(depth=10, ref=p + 1) == EINVAL and call(ops=o + 4) == EINVAL
    assert not b.any()
    assert emuhevc.emu_launch_count() == before
