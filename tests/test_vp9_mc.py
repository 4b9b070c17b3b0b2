"""CPU tier for VP9 motion compensation (VP9DSPContext's mc / smc tables, ffmpeg_b200/csrc/vp9mc.cu): the checker
(oracle/vp9mc_oracle.c) against the compiled reference (oracle/_ref/libffref_vp9dsp.so) member by member and on the decoder's batch
sequence, the filter tables, the fixture hashes, the layout marker, the ctypes mirrors, and vp9mc.cu itself, host code included, on the
stand-in CUDA runtime of tests/cuda_emu (the batch entry, sentinels, every table entry of every depth, and the refusals)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vp9mclib as vm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", vm.DEPTHS)
@pytest.mark.parametrize("cls", (0, 1, 2, 3), ids=("noise", "zero", "max", "extremes"))
def test_checker_mc_members_match_reference(depth, cls):
    """every mc entry (5 widths x 4 banks x put / avg x h x v) with every phase 0..15 in its filtered directions, heights 1..64"""
    seed = 100 + 13 * depth + cls
    ours = vm.run_members(cl.oracle(), "orc", seed, depth, cls, False)
    with vm.RefCheck() as rc:
        assert rc.same(ours, lambda: vm.run_members(vm.ref(), "ffref", seed, depth, cls, False))


@pytest.mark.parametrize("depth", vm.DEPTHS)
@pytest.mark.parametrize("cls", (0, 1, 2, 3), ids=("noise", "zero", "max", "extremes"))
def test_checker_smc_members_match_reference(depth, cls):
    """every smc entry over the step pairs of {1, 5, 8, 15, 16, 17, 20, 31, 32}^2 and all start phases"""
    seed = 200 + 13 * depth + cls
    assert {c[6:] for c in vm.smc_calls(seed)} == {(a, b) for a in vm.STEPS for b in vm.STEPS}
    ours = vm.run_members(cl.oracle(), "orc", seed, depth, cls, True)
    with vm.RefCheck() as rc:
        assert rc.same(ours, lambda: vm.run_members(vm.ref(), "ffref", seed, depth, cls, True))


@pytest.mark.parametrize("depth", vm.DEPTHS)
def test_sharp_bank_reaches_both_clip_bounds(depth):
    """on the alternating-extremes picture the sharp bank's sums leave the sample range on both sides, in the horizontal pass and in
    the vertical pass over the clipped intermediates, so a missing clip in either shows in the member tests"""
    pic, _ = vm.member_case(100 + 13 * depth + 3, depth, 3, False)
    F = vm.subpel_filters(cl.oracle(), "orc_vp9_subpel_filters")[2].astype(np.int64)
    maxv = (1 << depth) - 1
    p = pic.astype(np.int64)
    for m in (4, 8, 12):
        hs = (sum(F[m][k] * p[:, k:p.shape[1] - 7 + k] for k in range(8)) + 64) >> 7
        assert hs.min() < 0 and hs.max() > maxv, (m, hs.min(), hs.max())
        t = hs.clip(0, maxv)
        vs = (sum(F[m][k] * t[k:t.shape[0] - 7 + k] for k in range(8)) + 64) >> 7
        assert vs.min() < 0 and vs.max() > maxv, (m, vs.min(), vs.max())


@pytest.mark.parametrize("depth", vm.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_checker_batch_matches_decoder_sequence(depth, chroma):
    """the checker's clamped reads against the reference driver's edge tests + emulated_edge_mc windows + member calls: blocks at every
    edge and corner, windows wholly outside (positions up to 80 samples beyond the plane), compound ops whose slots name references of
    different size and step, compound ops with one full-pel and one fractional slot"""
    size = (100, 60) if chroma else (200, 120)
    for cls, scaled in ((0, True), (3, True), (0, False)):
        case = vm.batch_case(300 + depth + chroma + cls, 768, depth, *size, cls=cls, scaled=scaled)
        ops = case[3]
        mixed = ops[(ops["kind"] == vm.COMPOUND) & (ops["ref"][:, 0] != ops["ref"][:, 1])]
        assert len(mixed) > 50 or not scaled
        ours = vm.orc_batch(depth, *case)
        assert not np.array_equal(ours, case[2])
        with vm.RefCheck() as rc:
            assert rc.same(ours, lambda: vm.ref_batch(depth, *case))


def test_context_layout_matches_reference():
    """oracle/ref/ref_vp9dsp.c asserts at compile time that B200VP9DSPContext has VP9DSPContext's size, member offsets and
    function-pointer types: the marker proves the unit was compiled"""
    if not vm.have_ref():
        pytest.skip("oracle/_ref/libffref_vp9dsp.so not built")
    marker = C.c_char_p.in_dll(vm.ref(), "ffref_vp9dsp_layout_check")
    assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200VP9DSPContext matches")
    for depth in vm.DEPTHS:
        assert vm.ref().ffref_vp9_fpel_shared(depth) == 1


def kernel_filters():
    """the rows of vp9mc.cu's c_filters, parsed from the source: [4][16][8]"""
    txt = open(os.path.join(ROOT, "ffmpeg_b200", "csrc", "vp9mc.cu")).read()
    body = txt[txt.index("c_filters[4][16][8] = {"):]
    body = body[:body.index("};")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{([-0-9, ]+)\}", body)]
    return np.array(rows, np.int16).reshape(4, 16, 8)


def test_filter_tables():
    """the kernel's and the checker's 8-tap banks against the compiled reference's ff_vp9_subpel_filters (digest where it is not
    built); the kernel's bilinear bank is the 8-tap form of src[0] + ((m (src[1] - src[0]) + 8) >> 4)"""
    K, O = kernel_filters(), vm.subpel_filters(cl.oracle(), "orc_vp9_subpel_filters")
    assert np.array_equal(K[:3], O) and (O.sum(axis=2) == 128).all()
    with vm.RefCheck() as rc:
        assert rc.same(O, lambda: vm.subpel_filters(vm.ref(), "ffref_vp9_subpel_filters"))
    a, b = np.meshgrid(np.arange(0, 4096, 7), np.arange(0, 4096, 11))
    for m in range(16):
        assert list(K[3][m]) == [0, 0, 0, 128 - 8 * m, 8 * m, 0, 0, 0]
        assert np.array_equal((K[3][m][3] * a + K[3][m][4] * b + 64) >> 7, a + ((m * (b - a) + 8) >> 4))


def test_checker_reproduces_fixture():
    hs = vm.fixture_hashes()
    assert len(hs) == len(vm.DEPTHS) * 2
    for (depth, chroma), h in hs.items():
        assert vm.digest(vm.orc_batch(depth, *vm.fixture_case(depth, int(chroma)))) == h, (depth, chroma)


def test_ctypes_mirrors():
    from ffmpeg_b200._lib import VP9DSPContext, Vp9McOp, Vp9McRef
    from ffmpeg_b200 import vp9dsp
    assert C.sizeof(Vp9McOp) == vp9dsp.OP_DTYPE.itemsize == 40 and C.sizeof(Vp9McRef) == 32
    for name, _ in Vp9McOp._fields_:
        assert getattr(Vp9McOp, name).offset == vp9dsp.OP_DTYPE.fields[name][1], name
    assert C.sizeof(VP9DSPContext) == (96 + 160 + 40) * 8 and VP9DSPContext.mc.offset == 96 * 8 and VP9DSPContext.smc.offset == 256 * 8


# ---------------------------------------------------------------- vp9mc.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emuvp9():
    """libemuvp9.so: vp9mc.cu with its host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The kernel uses shared
    memory, __syncthreads and __syncwarp, so it runs an OS thread per CUDA thread of a block (emu.h's block launch), and __syncwarp
    becomes the warp's barrier."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vp9mc.cu", "tx_pfa.cu"):                           # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vp9mc.cu":
            assert t.count("extern __shared__ int16_t vp9_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { vp9_mc_kernel<") == 2
            t = t.replace("extern __shared__ int16_t vp9_smem[];", "int16_t *vp9_smem = (int16_t *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { vp9_mc_kernel<", "emu_cfg_launch(2, [&] { vp9_mc_kernel<")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        assert "<<<" not in t
        p = os.path.join(gen, "vp9_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuvp9.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_vp9_dsp_init.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp9_mc_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t]
    L.emu_launch_count.restype = C.c_uint64
    return L


def emu_batch(L, depth, planes, steps, dst, ops):
    d = dst.copy()
    ops = np.ascontiguousarray(ops)
    r = L.b200_vp9_mc_batch_device(None, depth, len(planes), C.cast(vm.ref_array(planes, steps), C.c_void_p), len(ops), ops.ctypes.data,
                                   d.ctypes.data, d.strides[0])
    assert r == 0
    return d


@pytest.mark.parametrize("depth", vm.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_emu_batch_vs_checker_and_fixture(emuvp9, depth, chroma):
    """the fixture batch through the library's entry: equal to the checker over the whole destination (the sentinels around and
    between the blocks unchanged) and to the reference's hash"""
    case = vm.fixture_case(depth, chroma)
    got = emu_batch(emuvp9, depth, *case)
    exp = vm.orc_batch(depth, *case)
    assert np.array_equal(got, exp)
    assert vm.digest(got) == vm.fixture_hashes()[(depth, bool(chroma))]
    sentinel = case[2][0, 0]
    assert (got == sentinel).sum() >= case[2].size - int((case[3]["w"].astype(int) * case[3]["h"]).sum())


def test_emu_unscaled_batch_vs_checker(emuvp9):
    """same-size references only (the mc table's 1-D, 2-D and full-pel entries), the extremes picture, run-of-ops CTAs"""
    case = vm.batch_case(31, 8200, 8, cls=3, scaled=False, cols=64)
    assert np.array_equal(emu_batch(emuvp9, 8, *case), vm.orc_batch(8, *case))


def test_emu_invalid_ops_write_nothing(emuvp9):
    """undefined kinds, banks and widths, a reference index beyond nrefs, h outside 1..64, phases above 15, odd offsets at 16 bit: nothing
    written; the valid ops of the same call are"""
    for depth in (8, 10):
        planes, steps, dst, ops = vm.batch_case(51, 16, depth)
        bad = ops.copy()
        bad["kind"][0], bad["kind"][1], bad["filter"][2], bad["filter"][3] = 2, 255, 4, 255
        bad["w"][4], bad["w"][5], bad["w"][6], bad["h"][7], bad["h"][8] = 0, 12, 65, 0, 65
        bad["ref"][9, 0], bad["kind"][10], bad["ref"][10, 1] = 8, 1, 200
        bad["mx"][11, 0], bad["my"][12, 0], bad["kind"][13], bad["my"][13, 1] = 16, 255, 1, 16
        if depth > 8:
            bad["dst_off"][14] += 1
        n = 15 if depth > 8 else 14
        assert np.array_equal(emu_batch(emuvp9, depth, planes, steps, dst, bad[:n]), dst)
        assert np.array_equal(vm.orc_batch(depth, planes, steps, dst, bad[:n]), dst)
        got = emu_batch(emuvp9, depth, planes, steps, dst, bad)
        assert np.array_equal(got, vm.orc_batch(depth, planes, steps, dst, bad)) and not np.array_equal(got, dst)
        # a slot the op does not use may hold anything
        single = ops.copy()
        single["kind"], single["ref"][:, 1], single["mx"][:, 1] = 0, 255, 255
        assert np.array_equal(emu_batch(emuvp9, depth, planes, steps, dst, single), vm.orc_batch(depth, planes, steps, dst, single))


def test_emu_every_table_entry(emuvp9):
    """every mc and smc entry at every depth through host pointers against the checker (every third call of the generators, which
    still takes every entry), and out-of-domain member arguments writing nothing"""
    from ffmpeg_b200._lib import VP9DSPContext
    from test_vp9_mc_gpu import check_members, run_ctx_mc, run_ctx_smc
    for depth in vm.DEPTHS:
        ctx = VP9DSPContext()
        assert emuvp9.b200_vp9_dsp_init(C.byref(ctx), depth) == 0
        check_members(ctx, depth, 70 + depth, 0 if depth != 10 else 3, stride=3)
    pic, dst0 = vm.member_case(1, 12, 0, True)
    for call in ((16, 1, 0, 1, 1, 0, 3, 3), (16, 1, 0, 1, 1, 65, 3, 3), (16, 1, 1, 1, 1, 8, 16, 3), (16, 1, 0, 1, 1, 8, 3, -1)):
        assert np.array_equal(run_ctx_mc(ctx, call, pic, dst0), dst0), call
    for call in ((16, 1, 0, 8, 3, 3, 0, 16), (16, 1, 1, 8, 3, 3, 16, 33), (8, 3, 0, 8, 3, 16, 16, 16)):
        assert np.array_equal(run_ctx_smc(ctx, call, pic, dst0), dst0), call


def test_emu_member_pattern(emuvp9):
    """mc and smc filled completely, every other member NULL; the four full-pel entries of a size and put / avg are one function"""
    from ffmpeg_b200._lib import VP9DSPContext
    ctx = VP9DSPContext()
    assert emuvp9.b200_vp9_dsp_init(C.byref(ctx), 10) == 0
    words = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
    assert (words[:96] == 0).all() and (words[96:] != 0).all()
    mc = words[96:256].reshape(5, 4, 2, 2, 2)
    for i in range(5):
        for a in range(2):
            assert len(set(mc[i, :, a, 0, 0])) == 1
    assert len(set(words[96:])) == 5 * 2 + 5 * 4 * 2 * 3 + 40


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emuvp9):
    from ffmpeg_b200._lib import VP9DSPContext
    for L in (prodlib, emuvp9):
        ctx = VP9DSPContext()
        for depth in (0, 7, 9, 11, 13, 14, 16):
            assert L.b200_vp9_dsp_init(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_vp9_dsp_init(None, 8) == EINVAL


def test_batch_refusals(prodlib, emuvp9):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    from ffmpeg_b200._lib import Vp9McRef
    b = np.zeros(8192, np.uint8)
    p = b.ctypes.data
    ops = np.zeros(1, vm.OP_DTYPE)
    ops["w"] = ops["h"] = 4
    o = ops.ctypes.data
    before = emuvp9.emu_launch_count()
    for L in (prodlib, emuvp9):
        def call(depth=8, nrefs=1, n=1, ops=o, dst=p + 64, ds=64, refs=True, data=p + 4096, rs=64, w=16, h=16, dx=16, dy=16, last=None):
            arr = (Vp9McRef * 8)(*[Vp9McRef(data, rs, w, h, dx, dy)] * 8)
            if last is not None:
                arr[nrefs - 1] = Vp9McRef(*last)
            return L.b200_vp9_mc_batch_device(None, depth, nrefs, C.cast(arr, C.c_void_p) if refs else None, n, ops, dst, ds)
        assert call(n=0) == 0 and call(n=0, ops=None, dst=None, refs=False) == 0
        assert call(n=-1) == EINVAL and call(nrefs=0) == EINVAL and call(nrefs=9) == EINVAL and call(nrefs=-1) == EINVAL
        for depth in (0, 7, 9, 11, 13, 14, 16):
            assert call(depth=depth) == EINVAL, depth
        assert call(w=0) == EINVAL and call(h=0) == EINVAL and call(w=-5) == EINVAL and call(data=None) == EINVAL
        for step in (0, -1, 33):
            assert call(dx=step) == EINVAL and call(dy=step) == EINVAL
        assert call(nrefs=8, last=(p + 4096, 64, 16, 16, 16, 40)) == EINVAL       # the last of eight references
        assert call(depth=10, ds=63) == EINVAL and call(depth=12, rs=65) == EINVAL and call(depth=10, data=p + 4097) == EINVAL
        for k in ("ops", "dst"):
            assert call(**{k: None}) == EINVAL, k
        assert call(refs=False) == EINVAL
        assert call(depth=10, dst=p + 65) == EINVAL and call(ops=o + 4) == EINVAL
    assert not b.any()
    assert emuvp9.emu_launch_count() == before
