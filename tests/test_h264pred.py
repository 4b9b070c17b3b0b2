"""CPU tier for H.264 intra prediction (H264PredContext, ffmpeg_b200/csrc/h264pred.cu): the checker (oracle/h264pred_oracle.c) against
the compiled reference (oracle/_ref/libffref_h264pred.so) and the fixture hashes, the product's init and argument checks, and h264pred.cu itself, host code included, on
the stand-in CUDA runtime of tests/cuda_emu (both batched entries and every drop-in member against the checker)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import h264predlib as hp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
DEPTHS = (8, 9, 10, 12, 14)
CODEC_H264, CODEC_SVQ3, CODEC_RV40, CODEC_VP8, CODEC_VP7 = 27, 23, 69, 139, 178
EINVAL, ENOSYS = -22, -38
MEMBERS = [("pred4x4", 15), ("pred8x8l", 12), ("pred8x8", 11), ("pred16x16", 9), ("pred4x4_add", 2), ("pred8x8l_add", 2),
           ("pred8x8l_filter_add", 2), ("pred8x8_add", 3), ("pred16x16_add", 3)]


def fixture_hashes():
    out = {}
    for line in open(os.path.join(ROOT, "tests", "golden", "h264pred_hashes.txt")):
        d, idc, what, h = line.split()
        out[(int(d), int(idc), what == "add")] = h
    return out


def digest(pic, coef):
    return hashlib.sha256(np.ascontiguousarray(pic).tobytes() + np.ascontiguousarray(coef).tobytes()).hexdigest()


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("idc", (0, 1, 2, 3))
@pytest.mark.parametrize("add", (False, True), ids=("pred", "add"))
def test_checker_matches_reference(depth, idc, add):
    """every member of ff_h264_pred_init(H.264, depth, idc) over fresh seeded cases (idc 0 and 3 check the 8x8 / 8x16 choice)"""
    n = 3 * len(hp.PRED_CLASSES) * len(hp.h264pred_combos(idc, add))
    case = hp.h264pred_case(3000 + 17 * depth + 5 * idc + add, n, depth, idc, add)
    ours = hp.orc_h264pred(depth, idc, add, *case)
    assert not np.array_equal(ours[0], case[0])
    if add:
        assert not np.array_equal(ours[1], case[4])
    with hp.RefCheck() as rc:
        assert rc.same(list(ours), lambda: list(hp.ref_h264pred(depth, idc, add, *case)))


def test_context_layout_matches_reference():
    """oracle/ref/ref_h264pred.c asserts at compile time that B200H264PredContext has H264PredContext's size, member offsets and
    function-pointer types, and that B200_CODEC_ID_H264 is AV_CODEC_ID_H264: the marker proves the unit was compiled"""
    if not hp.have_ref():
        pytest.skip("oracle/_ref/libffref_h264pred.so not built")
    marker = C.c_char_p.in_dll(hp.ref(), "ffref_h264pred_layout_check")
    assert C.string_at(C.addressof(marker)).startswith(b"b200dsp.h B200H264PredContext matches")


def test_checker_reproduces_fixture():
    hs = fixture_hashes()
    assert len(hs) == len(DEPTHS) * 2 * 2
    for (depth, idc, add), h in hs.items():
        assert digest(*hp.orc_h264pred(depth, idc, add, *hp.h264pred_fixture_case(depth, idc, add))) == h, (depth, idc, add)


# ---------------------------------------------------------------- h264pred.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emupred():
    """libemupred.so: h264pred.cu with its host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h.  The prediction
    kernel uses shared memory and __syncthreads, so it runs one OS thread per CUDA thread of a block (emu.h's block launch)."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("h264pred.cu", "tx_pfa.cu"):                       # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "h264pred.cu":
            assert t.count("extern __shared__ int pred_smem[];") == 1 and t.count("emu_cfg_launch(0, [&] { h264_pred_kernel<") == 2
            t = t.replace("extern __shared__ int pred_smem[];", "int *pred_smem = (int *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { h264_pred_kernel<", "emu_cfg_launch(2, [&] { h264_pred_kernel<")
        assert "<<<" not in t
        p = os.path.join(gen, "pred_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemupred.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_h264_pred_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.b200_h264_pred_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int64] + [C.c_void_p] * 4 + [C.c_ssize_t]
    L.b200_h264_pred_add_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int64] + [C.c_void_p] * 4 + [C.c_ssize_t] + [C.c_void_p] * 2
    return L


def run_batch(L, depth, add, pic, kinds, flags, off, coef, coef_off, dev=None):
    """one batched call on host-addressable buffers (the stand-in runtime's device memory is host memory)"""
    d, cf = pic.copy(), coef.copy()
    if add:
        r = L.b200_h264_pred_add_batch_device(dev, depth, len(kinds), kinds.ctypes.data, flags.ctypes.data, d.ctypes.data, off.ctypes.data,
                                              d.strides[0], cf.ctypes.data, coef_off.ctypes.data)
    else:
        r = L.b200_h264_pred_batch_device(dev, depth, len(kinds), kinds.ctypes.data, flags.ctypes.data, d.ctypes.data, off.ctypes.data, d.strides[0])
    assert r == 0
    return d, cf


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("idc", (1, 2))
def test_emu_batch_entries(emupred, depth, idc):
    """both batched entries on a whole seeded picture (every table, mode and flags value, every content class) against the checker
    and the reference's fixture hashes: samples outside each op's block untouched, coefficients cleared by the add forms"""
    hs = fixture_hashes()
    for add in (False, True):
        case = hp.h264pred_fixture_case(depth, idc, add)
        got = run_batch(emupred, depth, add, *case)
        exp = hp.orc_h264pred(depth, idc, add, *case)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (depth, idc, add)
        assert digest(*got) == hs[(depth, idc, add)]


def test_emu_invalid_kinds_change_nothing(emupred):
    """kinds naming members the reference leaves NULL (or no table at all) leave samples and coefficients alone"""
    bad_pred = [(0, 12), (0, 15), (1, 12), (2, 11), (3, 15), (4, 7), (4, 8), (5, 0), (15, 15)]
    bad_add = [(0, 2), (1, 3), (2, 2), (3, 0), (4, 0), (5, 0), (5, 3), (6, 1), (15, 15)]
    for depth in (8, 10):
        for add, bad in ((False, bad_pred), (True, bad_add)):
            pic, kinds, flags, off, coef, coef_off = hp.h264pred_case(77, len(bad), depth, 1, add)
            kinds = np.array([(t << 4) | m for t, m in bad], np.uint8)
            got = run_batch(emupred, depth, add, pic, kinds, flags, off, coef, coef_off)
            assert np.array_equal(got[0], pic) and np.array_equal(got[1], coef), (depth, add)


def member_of(table, mode, idc, add):
    """(H264PredContext member name, index) that batched (table, mode) stands for"""
    if add:
        return [("pred4x4_add", mode), ("pred8x8l_add", mode), ("pred8x8l_filter_add", mode), ("pred8x8_add", mode), ("pred8x8_add", mode),
                ("pred16x16_add", mode)][table]
    return [("pred4x4", mode), ("pred8x8l", mode), ("pred8x8", mode), ("pred8x8", mode), ("pred16x16", mode)][table]


def run_members(ctx, depth, idc, add, pic, kinds, flags, off, coef, coef_off, field=False):
    """every op of a case through the H264PredContext member it names, with HOST pointers: pred4x4's topright from a separate buffer,
    pred8x8l's flags as the decoder's 0x8000 / 0x4000, the 8x8 / 8x16 / 16x16 add forms with the decoder's block_offset table (frame: the
    picture's line size; field: twice the line size, the table of block_offset[48..] relative to it)"""
    d, cf = pic.copy(), coef.copy()
    bps, stride = pic.itemsize, pic.strides[0]
    st = 2 * stride if field else stride
    bo = hp.pred_block_offsets(st, bps)
    for i in range(len(kinds)):
        t, m = int(kinds[i]) >> 4, int(kinds[i]) & 15
        name, idx = member_of(t, m, idc, add)
        fn = getattr(ctx, name)[idx]
        src = d.ctypes.data + int(off[i])
        if add:
            blk = cf.ctypes.data + int(coef_off[i]) * cf.itemsize
            if name == "pred8x8l_filter_add":
                fn(src, blk, 0x8000 if flags[i] & 1 else 0, 0x4000 if flags[i] & 2 else 0, stride)
            elif name in ("pred8x8_add", "pred16x16_add"):
                fn(src, bo.ctypes.data, blk, st)
            else:
                fn(src, blk, stride)
        elif name == "pred4x4":
            tr = np.frombuffer(C.string_at(src + (4 if flags[i] & 2 else 3) * bps - stride, 4 * bps), pic.dtype).copy()
            if not flags[i] & 2:
                tr[:] = tr[0]
            fn(src, tr.ctypes.data, stride)
        elif name == "pred8x8l":
            fn(src, 0x8000 if flags[i] & 1 else 0, 0x4000 if flags[i] & 2 else 0, stride)
        else:
            fn(src, stride)
    return d, cf


def checker_field(depth, idc, pic, kinds, flags, off, coef, coef_off):
    """the checker on the field form: the same sub-block tables at twice the line size"""
    O = cl.oracle()
    O.orc_h264_pred.argtypes = [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t]
    d, cf = pic.copy(), coef.copy()
    st = 2 * pic.strides[0]
    bo = hp.pred_block_offsets(st, pic.itemsize)
    for i in range(len(kinds)):
        t, m = int(kinds[i]) >> 4, int(kinds[i]) & 15
        table, tidc = hp.ADD_TABLE_MAP[t]
        assert O.orc_h264_pred(depth, tidc or idc, table, m, d.ctypes.data + int(off[i]), None, 0,
                               cf.ctypes.data + int(coef_off[i]) * cf.itemsize, bo.ctypes.data, st) == 0
    return d, cf


def field_case(depth, idc):
    """the 8x8 / 8x16 / 16x16 add forms only, in cells tall enough for a field macroblock (32 picture rows + the row above)"""
    combos = [c for c in hp.h264pred_combos(idc, True) if c[0] >= 3]
    n = 4 * len(combos)
    pic, kinds, flags, off, coef, coef_off = hp.h264pred_case(4100 + depth + idc, 2 * n, depth, idc, True, cols=8)
    sel = np.arange(n) * 2                                      # one op per two cells: cell 2k and 2k + 8 (the one below) stay free
    rows = (np.arange(n) // 8) * 2
    off = ((rows * hp.PRED_CELL + 8) * pic.strides[0] + ((np.arange(n) % 8) * hp.PRED_CELL + 8) * pic.itemsize).astype(np.int64)
    kinds = np.array([(c[0] << 4) | c[1] for c in combos] * 4, np.uint8)
    return pic, kinds, np.zeros(n, np.uint8), off, coef[sel], coef_off[:n]


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("idc", (1, 2))
def test_emu_dropin_members(emupred, depth, idc):
    """every member b200_h264_pred_init fills, called through the table with host pointers, against the checker; the member NULL
    pattern against the reference's"""
    from ffmpeg_b200._lib import H264PredContext
    ctx = H264PredContext()
    assert emupred.b200_h264_pred_init(C.byref(ctx), CODEC_H264, depth, idc) == 0
    for add in (False, True):
        case = hp.h264pred_case(4000 + depth + 3 * idc + add, len(hp.PRED_CLASSES) * len(hp.h264pred_combos(idc, add)), depth, idc, add)
        got = run_members(ctx, depth, idc, add, *case)
        exp = hp.orc_h264pred(depth, idc, add, *case)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (depth, idc, add)
    fc = field_case(depth, idc)
    got = run_members(ctx, depth, idc, True, *fc, field=True)
    exp = checker_field(depth, idc, *fc)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]) and not np.array_equal(got[0], fc[0])


def member_mask(ctx):
    return np.array([1 if getattr(ctx, name)[i] else 0 for name, n in MEMBERS for i in range(n)], np.uint8)


def test_emu_member_null_pattern(emupred):
    from ffmpeg_b200._lib import H264PredContext
    with hp.RefCheck() as rc:
        for depth in DEPTHS:
            for idc in (0, 1, 2, 3):
                ctx = H264PredContext()
                assert emupred.b200_h264_pred_init(C.byref(ctx), CODEC_H264, depth, idc) == 0
                ours = member_mask(ctx)
                assert ours.sum() == 12 + 12 + 11 + 7 + 2 + 2 + 2 + 2 + 2

                def theirs():
                    R = hp.ref()
                    R.ffref_h264_pred_members.argtypes = [C.c_int, C.c_int, C.c_void_p]
                    m = np.zeros(64, np.uint8)
                    assert R.ffref_h264_pred_members(depth, idc, m.ctypes.data) == len(ours)
                    return m[:len(ours)]
                assert rc.same(ours, theirs), (depth, idc)


# ---------------------------------------------------------------- refusals of the product library (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emupred):
    from ffmpeg_b200._lib import H264PredContext
    for L in (prodlib, emupred):
        ctx = H264PredContext()
        for cid in (CODEC_SVQ3, CODEC_RV40, CODEC_VP8, CODEC_VP7, 0):
            assert L.b200_h264_pred_init(C.byref(ctx), cid, 8, 1) == ENOSYS, cid
        for depth in (0, 7, 11, 13, 16):
            assert L.b200_h264_pred_init(C.byref(ctx), CODEC_H264, depth, 1) == ENOSYS, depth
        assert L.b200_h264_pred_init(None, CODEC_H264, 8, 1) == EINVAL
        assert L.b200_h264_pred_init(C.byref(ctx), CODEC_H264, 8, 4) == EINVAL
        assert L.b200_h264_pred_init(C.byref(ctx), CODEC_H264, 8, -1) == EINVAL


def test_batch_refusals(prodlib, emupred):
    b = np.zeros(64, np.uint8)
    p = b.ctypes.data
    for L in (prodlib, emupred):
        for add in (False, True):
            def call(depth, n, kinds=p, flags=p, pix=p, off=p, stride=16, coef=p, coef_off=p):
                if add:
                    return L.b200_h264_pred_add_batch_device(None, depth, n, kinds, flags, pix, off, stride, coef, coef_off)
                return L.b200_h264_pred_batch_device(None, depth, n, kinds, flags, pix, off, stride)
            assert call(8, 0) == 0 and call(8, 0, None, None, None, None) == 0
            assert call(8, -1) == EINVAL and call(8, 1, stride=-16) == EINVAL
            for depth in (0, 7, 11, 16):
                assert call(depth, 1) == EINVAL, depth
            assert call(10, 1, stride=17) == EINVAL and call(10, 1, pix=p + 1) == EINVAL
            for k in ("kinds", "flags", "pix", "off") + (("coef", "coef_off") if add else ()):
                assert call(8, 1, **{k: None}) == EINVAL, k
            assert not b.any()
