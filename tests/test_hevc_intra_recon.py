"""CPU tier for HEVC intra reconstruction of a whole picture (b200_hevc_intra_recon_picture_device, ffmpeg_b200/csrc/hevcintra.cu): the
checker (oracle/hevcintra_oracle.c) against the compiled reference (oracle/_ref/libffref_hevcintra.so: the reference's intra_pred and
residual members driven over all components in decode order) on generated pictures (luma only and 4:2:0 / 4:2:2 / 4:4:4, CTB 16 / 32 / 64
with sizes that are not CTB multiples, slices and tiles, constrained intra prediction, smoothing and strong smoothing on and off, every
TU kind and flag and TUs without residual, depths 8, 9, 10 and 12); the fixture hashes; the fixture pictures telling the decode order
apart from an order without dependencies; the layouts; and hevcintra.cu itself, host code included, on the stand-in CUDA runtime of
tests/cuda_emu (fixture pictures with sentinels, the per-level path of the batch entries on the same pictures, invalid ops, refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hevcintralib as hl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL = -22


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------- the checker against the reference
PICTURES = {   # name -> (depth, chroma_format_idc, W, H, log2_ctb, kwargs)
    "400-8-ctb16-slices": (8, 0, 200, 136, 4, dict(nslices=3)),
    "420-9-ctb32-tiles": (9, 1, 232, 120, 5, dict(tiles=(2, 2), nslices=2)),
    "420-12-ctb64-nosmooth": (12, 1, 200, 136, 6, dict(smoothing=False)),
    "422-10-ctb32-cip": (10, 2, 136, 72, 5, dict(cip=True, tiles=(2, 1))),
    "422-8-ctb16-nostrong": (8, 2, 200, 104, 4, dict(strong=False, nslices=2)),
    "444-12-ctb16-cip": (12, 3, 120, 88, 4, dict(cip=True, nslices=2)),
    "444-9-ctb64-tiles": (9, 3, 200, 136, 6, dict(tiles=(2, 2))),
    "420-10-ctb64-cip-sparse": (10, 1, 264, 136, 6, dict(cip=True, p_intra=0.4)),
    "400-12-ctb32-cip": (12, 0, 168, 104, 5, dict(cip=True, strong=False)),
    "422-9-ctb64-cbf": (9, 2, 200, 136, 6, dict(p_cbf=0.95, split=0.8)),
}


def picture_of(name, seed_base=100):
    depth, cfmt, W, H, l2, kw = PICTURES[name]
    return hl.picture(seed_base + list(PICTURES).index(name), depth, cfmt, W, H, l2, **kw)


@pytest.mark.parametrize("name", list(PICTURES))
def test_checker_matches_reference(name):
    """whole pictures in decode order, the reference's intra_pred and residual sequence TU by TU (sentinels included)"""
    p = picture_of(name)
    kinds = set(int(k) for k in p.ops["tu_kind"])
    assert hl.TU_NONE in kinds and len(kinds) >= 5, kinds
    ours = hl.orc_picture(p)
    assert not same(ours, p.framed())
    with hl.RefCheck() as rc:
        assert rc.same(ours, lambda: hl.ref_picture(p))


def test_pictures_cover_the_flags():
    """across the pictures: every TU kind, every residual flag, 4:2:2 pairs, every neighbour flag and both component kinds"""
    ops = np.concatenate([picture_of(n).ops for n in PICTURES])
    assert set(int(k) for k in ops["tu_kind"]) == {0, 1, 2, 3, 4, hl.TU_NONE}
    for bit in (1, 2, 4):
        assert (ops["tu_flags"] & bit).any()
    for bit in range(8):
        assert (ops["flags"] & (1 << bit)).any() and not (ops["flags"] & (1 << bit)).all()
    assert set(int(v) for v in ops["plane"]) == {0, 1, 2} and set(int(v) for v in ops["log2_size"]) == {2, 3, 4, 5}


@pytest.mark.parametrize("name", hl.FIXTURE_NAMES)
def test_fixture_hashes(name):
    """the checker gives the reference's hash on every fixture picture (sentinels included)"""
    assert hl.digest(hl.orc_picture(hl.fixture_case(name))) == hl.fixture_hashes()[name]


def test_fixture_is_the_reference_result():
    if not hl.have_ref():
        pytest.skip("the reference is not built here; test_fixture_hashes checks the stored hashes")
    for name in hl.FIXTURE_NAMES:
        assert hl.digest(hl.ref_picture(hl.fixture_case(name))) == hl.fixture_hashes()[name], name


@pytest.mark.parametrize("name", hl.FIXTURE_NAMES)
def test_fixtures_need_the_dependencies(name):
    """every fixture picture comes out differently when each op reads the planes as they were before the call: a missing wait shows"""
    p = hl.fixture_case(name)
    assert not same(hl.orc_picture(p, order=1), hl.orc_picture(p))


def test_layouts():
    """RECON_DTYPE = HevcIntraReconOp = B200HevcIntraReconOp (32 bytes, static_assert in the header)"""
    from ffmpeg_b200 import hevcdsp
    from ffmpeg_b200._lib import HevcIntraReconOp
    assert C.sizeof(HevcIntraReconOp) == hevcdsp.RECON_DTYPE.itemsize == 32
    for name, _ in HevcIntraReconOp._fields_:
        assert getattr(HevcIntraReconOp, name).offset == hevcdsp.RECON_DTYPE.fields[name][1], name
    hdr = open(os.path.join(ROOT, "include", "b200dsp.h")).read()
    assert 'static_assert(sizeof(B200HevcIntraReconOp) == 32, "B200HevcIntraReconOp is 32 bytes");' in hdr
    assert "#define B200_HEVC_TU_NONE 0xFF" in hdr and hevcdsp.TU_NONE == 0xFF


# ---------------------------------------------------------------- hevcintra.cu on the stand-in runtime
PROGRESS_EMU = """// ---- inter-warp progress (stand-in: the warps of a block are OS threads that run at once)
static inline int ld_acquire(const int *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline void st_release(int *p, int v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline unsigned long long globaltimer()
{
    return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
static inline void __nanosleep(unsigned) { std::this_thread::yield(); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
template <typename T> static inline T __ldcg(const T *p) { return *p; }
static inline int atomicMax(int *p, int v)
{
    int o = __atomic_load_n(p, __ATOMIC_RELAXED);
    while (o < v && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return o;
}
"""


@pytest.fixture(scope="module")
def emurecon():
    """libemuhevcintra.so: hevcintra.cu, hevcpred.cu and hevcidct.cu with their host code (the per-level path too), compiled with g++
    against tests/cuda_emu/fake/cuda_runtime.h.  The picture kernel's progress helpers (PTX) become host atomics and a real clock, its
    static shared arrays statics (blocks run one at a time), and every thread of a block is an OS thread, so the warps of a block wait
    on one another for real."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("hevcintra.cu", "hevcpred.cu", "hevcidct.cu", "tx_pfa.cu"):      # tx_pfa.cu: fake_device.cpp links it
        src = open(os.path.join(cs, f)).read()
        if f == "hevcintra.cu":
            a, b = src.index("// ---- inter-warp progress\n"), src.index("// ---- end of inter-warp progress")
            src = "#include <chrono>\n#include <thread>\n" + src[:a] + PROGRESS_EMU + src[b:]
        t = rewrite_launches(src)
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "hevcintra.cu":
            assert t.count("emu_cfg_launch(0, [&] { hevc_recon_kernel<") == 2 and "asm" not in t
            t = t.replace("emu_cfg_launch(0, [&] { hevc_recon_kernel<", "emu_cfg_launch(2, [&] { hevc_recon_kernel<")
            t = t.replace("__shared__ __align__(16)", "alignas(16) static").replace("__shared__", "static")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
        if f == "hevcpred.cu":
            t = t.replace("extern __shared__ int ipred_smem[];", "int *ipred_smem = (int *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_", "emu_cfg_launch(2, [&] { hevc_")
        if f == "hevcidct.cu":
            t = t.replace("extern __shared__ int4 hevc_tu_smem[];", "int4 *hevc_tu_smem = (int4 *)emu_smem;")
            t = t.replace("emu_cfg_launch(0, [&] { hevc_tu_kernel<", "emu_cfg_launch(2, [&] { hevc_tu_kernel<")
        assert "<<<" not in t
        p = os.path.join(gen, "hrecon_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuhevcintra.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_hevc_intra_recon_picture_device.argtypes = [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int64,
                                                                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int]
    L.b200_hevc_intra_timeouts.argtypes = [C.c_void_p, C.c_void_p]
    L.b200_hevc_intra_pred_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int]
    L.b200_hevc_transform_add_batch_device.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t]
    L.emu_launch_count.restype = C.c_uint64
    return L


def emu_picture(L, p, ops=None):
    """the picture entry on fresh framed planes (sentinels included); coef in a 16-byte aligned buffer, checked unchanged"""
    bufs = p.framed()
    ops = np.ascontiguousarray(p.ops if ops is None else ops)
    cbuf, caddr = hl._coef16(p.coef)
    before = cbuf.copy()
    arr = (C.c_void_p * 3)(*p.ptrs(bufs))
    m = None if p.map is None else np.ascontiguousarray(p.map)
    ls_y, ls_uv = p.strides(bufs)
    assert L.b200_hevc_intra_recon_picture_device(None, p.depth, p.cfmt, p.W, p.H, arr, ls_y, ls_uv, len(ops), ops.ctypes.data, caddr,
                                                  None if m is None else m.ctypes.data, 0 if m is None else m.strides[0], p.log2_min_pu) == 0
    assert np.array_equal(cbuf, before)
    return bufs


def emu_levels(L, p):
    """the per-level path on fresh framed planes: per plane and dependency level one prediction batch, then one residual batch"""
    bufs = p.framed()
    cbuf, caddr = hl._coef16(p.coef)
    m = None if p.map is None else np.ascontiguousarray(p.map)
    ptrs = p.ptrs(bufs)
    for c, io, idx in hl.level_batches(p):
        hs, vs = p.shifts(c)
        st = bufs[c].strides[0]
        assert L.b200_hevc_intra_pred_batch_device(None, p.depth, ptrs[c], st, p.W, p.H, hs, vs, len(io), io.ctypes.data,
                                                   None if m is None else m.ctypes.data, 0 if m is None else m.strides[0], p.log2_min_pu) == 0
        tu = hl.level_tu_ops(p, idx, st)
        if len(tu):
            assert L.b200_hevc_transform_add_batch_device(None, p.depth, len(tu), tu.ctypes.data, caddr, ptrs[c], st) == 0
    return bufs


def emu_timeouts(L):
    n = C.c_int64(-1)
    assert L.b200_hevc_intra_timeouts(None, C.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("name", hl.FIXTURE_NAMES)
def test_emu_picture_vs_checker_and_fixture(emurecon, name):
    """the fixture picture through the library's entry: equal to the checker over the whole framed planes (the sentinels unchanged)
    and to the reference's hash; no wait ran out"""
    p = hl.fixture_case(name)
    got = emu_picture(emurecon, p)
    assert same(got, hl.orc_picture(p))
    assert hl.digest(got) == hl.fixture_hashes()[name]
    assert emu_timeouts(emurecon) == 0


@pytest.mark.parametrize("name", ["420-8", "422-12-cip", "444-8-cip", "420-9-sparse"])
def test_emu_picture_vs_level_path(emurecon, name):
    """the one-call entry and the per-level path of the batch entries give the same planes, bit for bit"""
    p = hl.fixture_case(name)
    assert same(emu_picture(emurecon, p), emu_levels(emurecon, p))


def bad_ops(p):
    """ops that write nothing: size, mode, kind out of range, DST4 on 8x8, x / y / coef_off unaligned, block or flagged neighbours
    outside the plane, plane index above the format's"""
    bad = np.zeros(14, p.ops.dtype)
    bad["log2_size"], bad["tu_kind"], bad["plane"], bad["x"], bad["y"] = 3, 0, 0, 8, 8
    bad["log2_size"][0], bad["log2_size"][1], bad["mode"][2], bad["tu_kind"][3] = 1, 6, 35, 5
    bad["tu_kind"][4] = 2                                       # DST4 on an 8x8
    bad["x"][5], bad["y"][6], bad["coef_off"][7] = 6, 10, 4
    bad["x"][8] = p.dims(0)[0] - 4                              # block past the right edge
    bad["y"][9] = p.dims(0)[1]                                  # below the plane
    bad["x"][10], bad["flags"][10] = 0, hl.INTRA_CAND_L          # left neighbours outside the plane
    bad["y"][11], bad["flags"][11] = 0, hl.INTRA_CAND_U
    bad["plane"][12] = 3 if p.cfmt else 1
    bad["coef_off"][13] = -8
    return bad


@pytest.mark.parametrize("name", ["420-8", "400-12"])
def test_emu_invalid_ops(emurecon, name):
    """invalid ops mixed into a picture write nothing and hold up no later op: the picture equals the one without them, and the
    checker agrees"""
    p = hl.fixture_case(name)
    rng = np.random.default_rng(5)
    bad = bad_ops(p)
    mixed = np.insert(p.ops, np.sort(rng.integers(0, len(p.ops), len(bad))), bad)
    want = hl.orc_picture(p)
    assert same(emu_picture(emurecon, p, mixed), want)
    assert same(hl.orc_picture(p, ops=mixed), want)
    only = emu_picture(emurecon, p, bad)
    assert same(only, p.framed())
    assert emu_timeouts(emurecon) == 0


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_refusals(prodlib, emurecon):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move); nops == 0
    returns 0 without a launch"""
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data + (-b.ctypes.data % 64)
    m = np.ones(4096, np.uint8)
    before = emurecon.emu_launch_count()
    for L in (prodlib, emurecon):
        def call(depth=8, cf=1, w=64, h=64, planes=(p, p + 8192, p + 12288), ls_y=64, ls_uv=32, nops=1, ops=p + 16384, coef=p + 32768,
                 mp=None, ms=0, pu=2):
            arr = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_hevc_intra_recon_picture_device(None, depth, cf, w, h, arr, ls_y, ls_uv, nops, ops, coef, mp, ms, pu)
        for depth in (0, 7, 11, 13, 16):
            assert call(depth=depth) == EINVAL, depth
        assert call(cf=-1) == EINVAL and call(cf=4) == EINVAL
        assert call(w=0) == EINVAL and call(h=0) == EINVAL and call(w=-5) == EINVAL and call(w=65537) == EINVAL
        assert call(planes=None) == EINVAL and call(planes=(p, None, p)) == EINVAL and call(planes=(None, p, p)) == EINVAL
        assert call(nops=-1) == EINVAL and call(nops=(1 << 30) + 1) == EINVAL
        assert call(ops=None) == EINVAL and call(coef=None) == EINVAL and call(ops=p + 16392) == EINVAL and call(coef=p + 32776) == EINVAL
        assert call(ls_y=60) == EINVAL and call(ls_uv=28) == EINVAL and call(ls_y=66) == EINVAL and call(cf=3, ls_uv=32) == EINVAL
        assert call(depth=10, ls_y=128, ls_uv=60) == EINVAL and call(depth=10, ls_y=124, ls_uv=64) == EINVAL
        assert call(planes=(p + 2, p + 8192, p + 12288)) == EINVAL and call(depth=10, ls_y=128, ls_uv=64, planes=(p, p + 8196, p + 12288)) == EINVAL
        assert call(mp=m.ctypes.data, ms=15) == EINVAL and call(mp=m.ctypes.data, ms=16, pu=1) == EINVAL
        assert call(mp=m.ctypes.data, ms=16, pu=7) == EINVAL
        assert call(nops=0, ops=None, coef=None) == 0
        assert call(nops=0, cf=0, planes=(p, None, None), ops=None, coef=None) == 0
        assert L.b200_hevc_intra_timeouts(None, None) == EINVAL
    assert not b.any()
    assert emurecon.emu_launch_count() == before
