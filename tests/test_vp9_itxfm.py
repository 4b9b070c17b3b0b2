"""CPU tier for VP9 inverse transforms (VP9DSPContext's itxfm_add members, ffmpeg_b200/csrc/vp9itxfm.cu): the checker
(oracle/vp9itxfm_oracle.c) against the compiled reference (oracle/_ref/libffref_vp9itxfm.so) member by member and on the decoder's
residual sequence, the fixture hashes, the layout marker, the ctypes mirror, and vp9itxfm.cu itself, host code included, on the stand-in
CUDA runtime of tests/cuda_emu (fixture batches with sentinels, every member at every depth, invalid ops, the init's table, refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vp9itxfmlib as vt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", vt.DEPTHS)
@pytest.mark.parametrize("cls", vt.CLASSES)
def test_checker_members_match_reference(depth, cls):
    """all 20 members, four calls each: the destination (sentinels around the block included) and the coefficient buffer the member
    leaves behind (all zero, or only block[0] cleared on the DC-only path)"""
    seed = 100 + 17 * depth + vt.CLASSES.index(cls)
    ours = vt.run_members(cl.oracle(), "orc", seed, depth, cls)
    with vt.RefCheck() as rc:
        assert rc.same(ours, lambda: vt.run_members(vt.ref(), "ffref", seed, depth, cls))


def test_coefficient_classes_reach_their_paths():
    """extremes hold the storage type's limits at every depth; dcmix has eob 1 with other coefficients set; the DC-only path leaves
    them in place while the full path clears the block"""
    O = cl.oracle()
    for depth in vt.DEPTHS:
        info = np.iinfo(vt.cdtype(depth))
        ext = np.concatenate([c[3].ravel() for c in vt.member_calls(1, depth, "extremes")])
        assert ext.max() == info.max and ext.min() == info.min
        for tx, typ, eob, b, dst0 in vt.member_calls(2, depth, "dcmix"):
            assert eob == 1 and np.count_nonzero(b.ravel()[1:]) > 0
            _, left = vt.run_member(O, "orc_vp9_itxfm", depth, (tx, typ, eob, b, dst0))
            dc = tx == 3 or (tx < 3 and typ == 0)
            assert left.ravel()[0] == 0 and (np.array_equal(left.ravel()[1:], b.ravel()[1:]) if dc else not left.any())


@pytest.mark.parametrize("depth", vt.DEPTHS)
def test_checker_batch_matches_decoder_sequence(depth):
    """the checker's batch against the reference driver (the member on a copy of each op's coefficients), all classes mixed"""
    case = vt.batch_case(300 + depth, 600, depth, classes=vt.CLASSES)
    ours = vt.orc_batch(depth, *case)
    assert not np.array_equal(ours, case[0])
    with vt.RefCheck() as rc:
        assert rc.same(ours, lambda: vt.ref_batch(depth, *case))


def test_checker_reproduces_fixture():
    hs = vt.fixture_hashes()
    assert len(hs) == len(vt.DEPTHS) * len(vt.FIXTURE_CLASSES)
    for (depth, cls), h in hs.items():
        assert vt.digest(vt.orc_batch(depth, *vt.fixture_case(depth, cls))) == h, (depth, cls)


def test_context_layout_and_sharing_match_reference():
    """the B200VP9DSPContext layout marker of the VP9 reference build still matches, and the reference's itxfm_add table shares its
    pointers as the library's does: [3][*] one function, [4][*] one function, the 12 of [0..2] distinct"""
    import vp9mclib as vm
    if not (vm.have_ref() and vt.have_ref()):
        pytest.skip("oracle/_ref/libffref_vp9dsp.so / libffref_vp9itxfm.so not built")
    marker = C.c_char_p.in_dll(vm.ref(), "ffref_vp9dsp_layout_check")
    assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200VP9DSPContext matches")
    for depth in vt.DEPTHS:
        assert vt.ref().ffref_vp9_itxfm_shared(depth) == 1


def test_ctypes_mirror():
    from ffmpeg_b200._lib import Vp9TxOp, VP9DSPContext
    from ffmpeg_b200 import vp9dsp
    assert C.sizeof(Vp9TxOp) == vp9dsp.TX_DTYPE.itemsize == 24
    for name, _ in Vp9TxOp._fields_:
        assert getattr(Vp9TxOp, name).offset == vp9dsp.TX_DTYPE.fields[name][1], name
    assert VP9DSPContext.itxfm_add.offset == 60 * 8 and VP9DSPContext.loop_filter_8.offset == 80 * 8


# ---------------------------------------------------------------- vp9itxfm.cu on the stand-in runtime
def build_emu(name, text_fn=None):
    """lib<name>.so: vp9itxfm.cu (after text_fn, if given) and vp9mc.cu with their host code, compiled with g++ against
    tests/cuda_emu/fake/cuda_runtime.h.  The kernel uses shared memory and __syncthreads, so it runs an OS thread per CUDA thread of a
    block (emu.h's block launch)."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vp9itxfm.cu", "vp9mc.cu", "tx_pfa.cu"):             # vp9mc.cu: b200_vp9_dsp_init; tx_pfa.cu: fake_device.cpp links it
        src = open(os.path.join(cs, f)).read()
        if f == "vp9itxfm.cu" and text_fn:
            src = text_fn(src)
        t = rewrite_launches(src)
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vp9itxfm.cu":
            assert t.count("extern __shared__ int4 vp9_itx_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { vp9_itx_kernel<") == 2
            t = t.replace("extern __shared__ int4 vp9_itx_smem[];", "int4 *vp9_itx_smem = (int4 *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { vp9_itx_kernel<", "emu_cfg_launch(2, [&] { vp9_itx_kernel<")
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
    L.b200_vp9_dsp_init_itxfm.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp9_itxfm_add_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t]
    L.emu_launch_count.restype = C.c_uint64
    return L


@pytest.fixture(scope="module")
def emuitx():
    return build_emu("emuvp9itx")


def emu_batch(L, depth, dst, coef, ops):
    d, c = dst.copy(), np.ascontiguousarray(coef)
    before = c.copy()
    ops = np.ascontiguousarray(ops)
    assert L.b200_vp9_itxfm_add_batch_device(None, depth, len(ops), ops.ctypes.data, c.ctypes.data, d.ctypes.data, d.strides[0]) == 0
    assert np.array_equal(c, before)                                 # coef is read only
    return d


@pytest.mark.parametrize("depth", vt.DEPTHS)
@pytest.mark.parametrize("cls", vt.FIXTURE_CLASSES)
def test_emu_batch_vs_checker_and_fixture(emuitx, depth, cls):
    """the fixture batch through the library's entry: equal to the checker over the whole destination (the sentinels around and
    between the blocks unchanged) and to the reference's hash"""
    case = vt.fixture_case(depth, cls)
    got = emu_batch(emuitx, depth, *case)
    assert np.array_equal(got, vt.orc_batch(depth, *case))
    assert vt.digest(got) == vt.fixture_hashes()[(depth, cls)]


@pytest.mark.parametrize("depth", vt.DEPTHS)
def test_emu_mixed_classes_vs_checker(emuitx, depth):
    """noise and eob-1-with-other-coefficients blocks, every member, CTAs of several ops"""
    case = vt.batch_case(40 + depth, 1200, depth, classes=("noise", "dcmix", "extremes"))
    assert np.array_equal(emu_batch(emuitx, depth, *case), vt.orc_batch(depth, *case))


def check_members(ctx, depth, seed, cls, per=2):
    """every member of the context through host pointers against the checker: destination and coefficients left behind"""
    from ffmpeg_b200.vp9dsp import VP9_ITXFM_FUNC
    O = cl.oracle()
    for call in vt.member_calls(seed, depth, cls, per):
        tx, typ, eob, b, dst0 = call
        d, blk = dst0.copy(), np.ascontiguousarray(b.copy())
        p = d.ctypes.data + vt.MARGIN * d.strides[0] + vt.MARGIN * d.itemsize
        VP9_ITXFM_FUNC(ctx.itxfm_add[tx][typ])(p, d.strides[0], blk.ctypes.data, eob)
        ed, eb = vt.run_member(O, "orc_vp9_itxfm", depth, call)
        assert np.array_equal(d, ed) and np.array_equal(blk, eb), (depth, cls, tx, typ, eob)


def test_emu_every_member(emuitx):
    """every member at every depth, each coefficient class"""
    from ffmpeg_b200._lib import VP9DSPContext
    for depth in vt.DEPTHS:
        ctx = VP9DSPContext()
        assert emuitx.b200_vp9_dsp_init_itxfm(C.byref(ctx), depth) == 0
        for cls in vt.CLASSES:
            check_members(ctx, depth, 70 + depth, cls, per=1)


def test_emu_invalid_ops_write_nothing(emuitx):
    """tx > 4, type > 3, coef_off not a multiple of 16, dst_off not a multiple of 4 samples: nothing written; the valid ops of the
    same call are"""
    for depth in (8, 10):
        dst, coef, ops = vt.batch_case(51, 16, depth)
        bad = ops.copy()
        bad["tx"][0], bad["tx"][1], bad["type"][2], bad["type"][3] = 5, 255, 4, 255
        bad["coef_off"][4] += 8
        bad["coef_off"][5] += 1
        bad["dst_off"][6] += 2 * dst.itemsize
        bad["dst_off"][7] += dst.itemsize
        assert np.array_equal(emu_batch(emuitx, depth, dst, coef, bad[:8]), dst)
        assert np.array_equal(vt.orc_batch(depth, dst, coef, bad[:8]), dst)
        got = emu_batch(emuitx, depth, dst, coef, bad)
        assert np.array_equal(got, vt.orc_batch(depth, dst, coef, bad)) and not np.array_equal(got, dst)


def table_words(ctx):
    return np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)


def test_emu_init_sets_exactly_the_table(emuitx):
    """on top of b200_vp9_dsp_init's context the init sets the 20 itxfm_add words and nothing else, with the reference's sharing:
    [3][*] one function, [4][*] one function, the twelve of [0..2] distinct; the depths' functions differ"""
    from ffmpeg_b200._lib import VP9DSPContext
    seen = set()
    for depth in vt.DEPTHS:
        ctx = VP9DSPContext()
        assert emuitx.b200_vp9_dsp_init(C.byref(ctx), depth) == 0
        w0 = table_words(ctx).copy()
        assert (w0[60:80] == 0).all()
        assert emuitx.b200_vp9_dsp_init_itxfm(C.byref(ctx), depth) == 0
        w1 = table_words(ctx)
        changed = np.nonzero(w0 != w1)[0]
        assert list(changed) == list(range(60, 80))
        t = w1[60:80].reshape(5, 4)
        assert len(set(t[3])) == 1 and len(set(t[4])) == 1 and len(set(t[:3].ravel())) == 12 and len(set(t.ravel())) == 14
        seen |= set(t.ravel())
    assert len(seen) == 3 * 14


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emuitx):
    from ffmpeg_b200._lib import VP9DSPContext
    for L in (prodlib, emuitx):
        ctx = VP9DSPContext()
        for depth in (0, 7, 9, 11, 13, 14, 16):
            assert L.b200_vp9_dsp_init_itxfm(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_vp9_dsp_init_itxfm(None, 8) == EINVAL
        assert not table_words(ctx).any()


def test_batch_refusals(prodlib, emuitx):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move)"""
    b = np.zeros(8192, np.uint8)
    p = b.ctypes.data + (-b.ctypes.data % 64)
    ops = np.zeros(1, vt.TX_DTYPE)
    o = ops.ctypes.data
    before = emuitx.emu_launch_count()
    for L in (prodlib, emuitx):
        def call(depth=8, n=1, ops=o, coef=p + 1024, dst=p + 4096, ds=64):
            return L.b200_vp9_itxfm_add_batch_device(None, depth, n, ops, coef, dst, ds)
        assert call(n=0) == 0 and call(n=0, ops=None, coef=None, dst=None) == 0
        assert call(n=-1) == EINVAL
        for depth in (0, 7, 9, 11, 13, 14, 16):
            assert call(depth=depth) == EINVAL, depth
        for k in ("ops", "coef", "dst"):
            assert call(**{k: None}) == EINVAL, k
        assert call(ops=o + 4) == EINVAL and call(coef=p + 1024 + 8) == EINVAL and call(dst=p + 4096 + 2) == EINVAL
        assert call(depth=10, dst=p + 4096 + 4) == EINVAL and call(ds=62) == EINVAL and call(depth=12, ds=68) == EINVAL
    assert not b.any()
    assert emuitx.emu_launch_count() == before
