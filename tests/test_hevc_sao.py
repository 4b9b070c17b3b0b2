"""CPU tier for HEVC sample adaptive offset (HEVCDSPContext's SAO members and b200_hevc_sao_plane_device, ffmpeg_b200/csrc/hevcsao.cu):
the checker (oracle/hevcsao_oracle.c) against the compiled reference (oracle/_ref/libffref_hevcsao.so) member by member and against
the decoder's own loop filter (hevc/filter.c) on whole pictures, the order independence of the out-of-place form, the fixture hashes
and their outcome coverage, the ctypes mirrors, and hevcsao.cu itself, host code included, on the stand-in CUDA runtime of
tests/cuda_emu (planes, sentinels, every member, the refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hevcsaolib as hl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_checker_band_matches_reference(depth):
    """every left_class 0..31 plus negative and large ones, int16 offsets up to the extremes, samples at 0 and the maximum; separate
    buffers and in place (dst == src, equal strides), sentinels around the block; every band pointer of the reference"""
    cases = list(hl.band_cases(300 + depth, depth))
    for in_place in (False, True):
        ours = [hl.orc_band(depth, c, in_place=in_place) for c in cases]
        with hl.RefCheck() as rc:
            assert rc.same(ours, lambda: [hl.ref_band(depth, c, in_place=in_place, idx=k % 5) for k, c in enumerate(cases)])


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_checker_edge_matches_reference(depth):
    """every class at every width and every height 1..64, offset_val[0] non-zero, sentinels around dst"""
    cases = list(hl.edge_cases(400 + depth, depth))
    ours = [hl.orc_edge(depth, c) for c in cases]
    with hl.RefCheck() as rc:
        assert rc.same(ours, lambda: [hl.ref_edge(depth, c, idx=k % 5) for k, c in enumerate(cases)])


@pytest.mark.parametrize("depth", hl.DEPTHS)
@pytest.mark.parametrize("which", (0, 1))
def test_checker_restore_sweep_matches_reference(depth, which):
    """sao_edge_restore[which] over every eo_class x borders[4] (x the eight edge flags for [1]) x c_idx 0..2 with non-zero
    offset_val[0], looped in C on both sides at several sizes, digests compared (margins around dst included)"""
    ours = [hl.sweep(depth, which, None, w, h, 7 + w) for w, h in hl.RESTORE_SIZES]
    with hl.RefCheck() as rc:
        assert rc.same(np.array(ours, np.uint64),
                       lambda: np.array([hl.sweep(depth, which, hl.ref().ffref_hevc_sao_restore_fn(depth, which), w, h, 7 + w)
                                         for w, h in hl.RESTORE_SIZES], np.uint64))


PICTURES = [  # (name, W, H, kwargs) luma sizes not multiples of 64
    ("slices_lf", 200, 136, dict(nslices=4, lf_slices=(1,), pcm=False)),
    ("slices_nolf", 200, 136, dict(nslices=5, lf_slices=(0,), pcm=True)),
    ("tiles_lf", 232, 152, dict(nslices=3, tiles=(3, 2), lf_tiles=True, pcm=True)),
    ("tiles_nolf", 232, 152, dict(nslices=4, tiles=(2, 2), lf_tiles=False, pcm=True, scatter=0.3)),
]


@pytest.mark.parametrize("depth", hl.DEPTHS)
@pytest.mark.parametrize("cfmt", (0, 1, 2, 3), ids=("luma", "420", "422", "444"))
def test_checker_plane_is_the_decoder(depth, cfmt):
    """per component, the checker's plane from the derived records against the decoder's hevc/filter.c run over the whole picture (all
    components in one run) at CTB sizes 16, 32 and 64: slices with and without loop_filter_across_slices, tiles with and without
    loop_filter_across_tiles, PCM / bypass maps marked in every quadrant of the chroma CTBs, NONE CTBs next to BAND and EDGE ones"""
    for log2_ctb in (4, 5, 6):
        for k, (name, W, H, kw) in enumerate(PICTURES):
            p = hl.picture_case(1000 + 31 * depth + 7 * cfmt + 3 * log2_ctb + k, depth, W, H, log2_ctb, cfmt, **kw)
            ours = []
            for c in range(len(p.planes)):
                W_, H_, _, _ = hl.comp_geometry(p, c)
                ours.append(hl.inner(hl.orc_plane(p, c), H_, W_))
                assert not np.array_equal(ours[-1], p.planes[c])
            with hl.RefCheck() as rc:
                assert rc.same(ours, lambda: hl.ref_picture(p)), (name, log2_ctb)


@pytest.mark.parametrize("cfmt", (0, 1, 2), ids=("luma", "420", "422"))
def test_checker_plane_order_does_not_matter(cfmt):
    """CTBs visited in raster and in reverse order give the same plane: the out-of-place form reads only the deblocked plane"""
    for depth in (8, 10):
        p = hl.picture_case(77 + depth + cfmt, depth, 232, 152, 5, cfmt, nslices=4, tiles=(2, 2), lf_tiles=False, pcm=True, scatter=0.2)
        for c in range(len(p.planes)):
            assert np.array_equal(hl.orc_plane(p, c), hl.orc_plane(p, c, reverse=True))


def test_fixture_reaches_every_outcome_and_matches():
    """the fixture planes: the checker reproduces the stored hashes of the reference's result, and between luma and chroma they reach
    every outcome (band, each edge class, border, each unfilterable edge and corner, each corner save, keep applied and keep
    skipped by the chroma quirk, clip at 0 and at the maximum)"""
    hs = hl.fixture_hashes()
    assert len(hs) == len(hl.DEPTHS) * 2
    for depth in hl.DEPTHS:
        assert hl.fixture_plane_hashes(depth) == {"luma": hs[(depth, "luma")], "chroma420": hs[(depth, "chroma420")]}
        cnt = hl.outcome_counts(hl.fixture_case(depth), [0, 1])
        assert all(v > 0 for v in cnt.values()), (depth, cnt)


def test_fixture_is_the_reference_result():
    if not hl.have_ref():
        pytest.skip("the reference is not built here; test_fixture_reaches_every_outcome_and_matches checks the stored hashes")
    for depth in hl.DEPTHS:
        p = hl.fixture_case(depth)
        got = hl.ref_picture(p)
        for c, name in ((0, "luma"), (1, "chroma420")):
            W, H, _, _ = hl.comp_geometry(p, c)
            assert hl.digest(hl.framed(got[c], depth)) == hl.fixture_hashes()[(depth, name)]


def test_ctypes_mirrors():
    from ffmpeg_b200._lib import HevcSaoCtb, SAOParams
    from ffmpeg_b200 import hevcdsp
    assert C.sizeof(HevcSaoCtb) == hevcdsp.SAO_DTYPE.itemsize == 16
    for name, _ in HevcSaoCtb._fields_:
        assert getattr(HevcSaoCtb, name).offset == hevcdsp.SAO_DTYPE.fields[name][1], name
    assert C.sizeof(SAOParams) == 148
    offs = {"offset_abs": 0, "offset_sign": 48, "band_position": 96, "eo_class": 100, "offset_val": 112, "type_idx": 142}
    for name, off in offs.items():
        assert getattr(SAOParams, name).offset == off, name


# ---------------------------------------------------------------- hevcsao.cu on the stand-in runtime
@pytest.fixture(scope="module")
def emusao():
    """libemuhevcsao.so: hevcsao.cu with its host code, compiled with g++ against tests/cuda_emu/fake/cuda_runtime.h (the plain kernel
    runs its threads one after the other)"""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("hevcsao.cu", "tx_pfa.cu"):                          # tx_pfa.cu: fake_device.cpp links against it
        t = rewrite_launches(open(os.path.join(cs, f)).read())
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "hevcsao.cu":
            assert t.count("emu_cfg_launch(0, [&] { hevc_sao_kernel<") == 2
        assert "<<<" not in t
        p = os.path.join(gen, "sao_" + f[:-3] + ".cpp")
        open(p, "w").write(t)
        srcs.append(p)
    so = os.path.join(gen, "libemuhevcsao.so")
    cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
    r = subprocess.run([cxx, "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-ffp-contract=off", "-w", "-D__host__=", "-I" + os.path.join(EMU, "fake"),
                        "-I" + cs, "-I" + os.path.join(ROOT, "include"), "-I" + EMU] + srcs + [os.path.join(EMU, "fake_device.cpp"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.b200_hevc_dsp_init_sao.argtypes = [C.c_void_p, C.c_int]
    L.b200_hevc_sao_plane_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int]
    L.emu_launch_count.restype = C.c_uint64
    L.b200_last_error.restype = C.c_char_p
    return L


def lib_plane(L, p, c, rec=None, keep="auto"):
    """component c through the library's plane entry: the whole sentinel-framed dst buffer; src, records and keep map unchanged"""
    W, H, hs, vs = hl.comp_geometry(p, c)
    g = hl.records(p, c, garbage_seed=5 + c) if rec is None else rec
    k = hl.keep_map(p) if keep == "auto" else keep
    src = hl.framed(p.planes[c], p.depth)
    dst = np.full_like(src, hl.sentinel(p.depth))
    s0, g0, k0 = src.copy(), g.copy(), None if k is None else k.copy()
    assert L.b200_hevc_sao_plane_device(None, p.depth, hl._ptr(dst), dst.strides[0], hl._ptr(src), src.strides[0], W, H, p.log2_ctb, hs, vs,
                                        g.ctypes.data, g.shape[1], None if k is None else k.ctypes.data, 0 if k is None else k.shape[1],
                                        p.log2_pu) == 0
    assert np.array_equal(src, s0) and np.array_equal(g, g0) and (k is None or np.array_equal(k, k0))
    return dst


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_emu_plane_vs_checker_and_fixture(emusao, depth):
    """the fixture picture's luma and chroma planes (records with garbage in the padding, in `reserved` and in unknown flag bits)
    through the library's entry: equal to the checker over the whole framed buffer (sentinels unchanged) and to the stored hash"""
    p = hl.fixture_case(depth)
    for c, name in ((0, "luma"), (1, "chroma420")):
        got = lib_plane(emusao, p, c)
        assert np.array_equal(got, hl.orc_plane(p, c))
        assert hl.digest(got) == hl.fixture_hashes()[(depth, name)]


@pytest.mark.parametrize("cfmt", (0, 1, 2, 3), ids=("luma", "420", "422", "444"))
def test_emu_plane_shapes(emusao, cfmt):
    """CTB sizes 16 / 32 / 64, odd plane sizes, no keep map, non-zero offset_val[0] (the picture-border value), and records with
    unknown types and edge classes above 3 (copied)"""
    for depth in (8, 10):
        for log2_ctb in (4, 5, 6):
            p = hl.picture_case(500 + depth + cfmt + log2_ctb, depth, 136 + 2 * log2_ctb, 72 + 2 * cfmt, log2_ctb, cfmt, nslices=3,
                                tiles=(2, 1), lf_tiles=False, pcm=log2_ctb != 5)
            for c in range(len(p.planes)):
                g = hl.records(p, c)
                g["offset_val"][:, :, 0] = np.random.default_rng(c).integers(-40, 41, g.shape)   # members honour any offset_val[0]
                g[0, 0]["type"], g[-1, 0]["type"] = 3, 255
                if p.cw > 1:
                    g[0, 1]["type"], g[0, 1]["cls"] = hl.SAO_EDGE, 4
                assert np.array_equal(lib_plane(emusao, p, c, rec=g), hl.orc_plane(p, c, rec=g)), (depth, log2_ctb, c)
    W, H = 37, 23                                                # odd luma plane, one partial CTB each way
    p = hl.picture_case(9, 10, W, H, 4, 0, nslices=1, pcm=False)
    assert np.array_equal(lib_plane(emusao, p, 0), hl.orc_plane(p, 0))


def _ctx(L, depth):
    from ffmpeg_b200._lib import HEVCDSPContext
    ctx = HEVCDSPContext()
    assert L.b200_hevc_dsp_init_sao(C.byref(ctx), depth) == 0
    return ctx


def check_members(ctx, depth, seed):
    """every band / edge pointer (in place and separate for band) and both restore sweeps through the context, against the checker"""
    for k, case in enumerate(hl.band_cases(seed, depth)):
        for in_place in (False, True):
            assert np.array_equal(hl.ctx_band(ctx, depth, case, in_place, idx=k % 5), hl.orc_band(depth, case, in_place=in_place)), (k, in_place)
    for k, case in enumerate(hl.edge_cases(seed + 1, depth)):
        if k % 3 == 0:
            assert np.array_equal(hl.ctx_edge(ctx, depth, case, idx=k % 5), hl.orc_edge(depth, case)), (k, case[1:4])
    for which in (0, 1):
        for w, h in hl.RESTORE_SIZES[:3]:
            assert hl.sweep(depth, which, ctx.sao_edge_restore[which], w, h, 3) == hl.sweep(depth, which, None, w, h, 3), (which, w, h)


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_emu_every_member(emusao, depth):
    ctx = _ctx(emusao, depth)
    assert len(set(ctx.sao_band_filter)) == 1 and len(set(ctx.sao_edge_filter)) == 1
    assert ctx.sao_edge_restore[0] and ctx.sao_edge_restore[1] and ctx.sao_edge_restore[0] != ctx.sao_edge_restore[1]
    check_members(ctx, depth, 60 + depth)


def test_emu_restore_launches_nothing_and_domain(emusao):
    """the restore members launch nothing; c_idx outside 0..2 and sizes outside 1..64 write nothing (all members)"""
    from ffmpeg_b200 import hevcdsp as hd
    from ffmpeg_b200._lib import SAOParams
    ctx = _ctx(emusao, 10)
    before = emusao.emu_launch_count()
    for which in (0, 1):
        hl.sweep(10, which, ctx.sao_edge_restore[which], 16, 9, 5)
    assert emusao.emu_launch_count() == before
    src = np.arange(80 * 80, dtype=np.uint16).reshape(80, 80) & 1023
    dst = np.full((80, 80), 7, np.uint16)
    sao = SAOParams()
    sao.offset_val[0][0] = sao.offset_val[1][0] = sao.offset_val[2][0] = 9
    b = (C.c_int * 4)(1, 1, 1, 1)
    e = (C.c_uint8 * 4)(1, 1, 1, 1)
    for which in (0, 1):
        for c_idx, w, h in ((-1, 8, 8), (3, 8, 8), (0, 0, 8), (0, 8, 0), (0, 65, 8), (0, 8, 65)):
            hd.SAO_EDGE_RESTORE(ctx.sao_edge_restore[which])(dst.ctypes.data, src.ctypes.data, 160, 160, C.byref(sao), b, w, h, c_idx, e, e, e)
    off = np.array([3, 4, 5, 6, 7], np.int16)
    for w, h in ((0, 4), (4, 0), (65, 4), (4, 65), (-1, 4)):
        hd.SAO_BAND_FILTER(ctx.sao_band_filter[0])(dst.ctypes.data, src.ctypes.data, 160, 160, off.ctypes.data, 0, w, h)
        hd.SAO_EDGE_FILTER(ctx.sao_edge_filter[0])(dst.ctypes.data, src.ctypes.data + 400, 160, off.ctypes.data, 0, w, h)
    for eo in (-1, 4, 100):
        hd.SAO_EDGE_FILTER(ctx.sao_edge_filter[0])(dst.ctypes.data, src.ctypes.data + 400, 160, off.ctypes.data, eo, 8, 8)
    assert (dst == 7).all()
    assert emusao.emu_launch_count() == before
    assert b"eo_class" in emusao.b200_last_error()


def test_emu_init_sets_exactly_the_sao_members(emusao):
    """the twelve SAO pointers are set, every other member of a filled context stays as it was"""
    from ffmpeg_b200._lib import HEVCDSPContext
    ctx = HEVCDSPContext()
    C.memset(C.addressof(ctx), 0x11, C.sizeof(ctx))
    before = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64).copy()
    assert emusao.b200_hevc_dsp_init_sao(C.byref(ctx), 12) == 0
    words = np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)
    sao = np.zeros(len(words), bool)
    first = HEVCDSPContext.sao_band_filter.offset // 8
    sao[first:first + 12] = True
    assert (words[sao] != before[sao]).all() and np.array_equal(words[~sao], before[~sao])


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emusao):
    from ffmpeg_b200._lib import HEVCDSPContext
    for L in (prodlib, emusao):
        ctx = HEVCDSPContext()
        for depth in (0, 7, 11, 13, 14, 16):
            assert L.b200_hevc_dsp_init_sao(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_hevc_dsp_init_sao(None, 8) == EINVAL
        assert not any(bytes(ctx))


def test_plane_refusals(prodlib, emusao):
    """every B200_EINVAL case launches nothing and writes nothing, overlapping dst / src included"""
    mem = np.zeros(3 * 64 * 128 + 256, np.uint8)
    base = (mem.ctypes.data + 63) & ~63
    dst, src = base, base + 64 * 128
    g = np.full(4096, 0x3F, np.uint8)
    grid = (g.ctypes.data + 15) & ~15
    k = np.full(4096, 1, np.uint8)
    keep = k.ctypes.data
    before = emusao.emu_launch_count()
    for L in (prodlib, emusao):
        def call(depth=8, d=dst, ds=128, s=src, ss=128, W=64, H=64, l2=5, hs=0, vs=0, c=grid, cs=2, kp=None, ks=0, pu=2):
            return L.b200_hevc_sao_plane_device(None, depth, d, ds, s, ss, W, H, l2, hs, vs, c, cs, kp, ks, pu)
        for kw in ({"d": None}, {"s": None}, {"c": None}):
            assert call(**kw) == EINVAL, kw
        for depth in (0, 7, 11, 13, 16):
            assert call(depth=depth) == EINVAL, depth
        for W, H in ((0, 8), (8, 0), (-4, 8), (8, -1)):
            assert call(W=W, H=H) == EINVAL, (W, H)
        for l2 in (3, 7, 0, -1):
            assert call(l2=l2) == EINVAL, l2
        for hs, vs in ((2, 0), (0, 2), (-1, 0), (0, -1)):
            assert call(hs=hs, vs=vs) == EINVAL, (hs, vs)
        assert call(ds=63) == EINVAL and call(ss=63) == EINVAL and call(ds=-128) == EINVAL and call(ss=0) == EINVAL
        assert call(depth=10, ds=127, ss=128, W=32) == EINVAL and call(depth=10, d=dst + 1, W=32) == EINVAL
        assert call(depth=10, s=src + 1, W=32) == EINVAL and call(c=grid + 8) == EINVAL
        assert call(cs=1) == EINVAL and call(W=65, cs=2) == EINVAL and call(cs=-1) == EINVAL and call(hs=1, l2=4, W=64, cs=7) == EINVAL
        assert call(kp=keep, ks=16, pu=1) == EINVAL and call(kp=keep, ks=16, pu=5) == EINVAL and call(kp=keep, ks=15, pu=2) == EINVAL
        assert call(kp=keep, ks=7, pu=3, hs=1, W=32) == EINVAL
        assert call(s=dst) == EINVAL and call(s=dst + 63 * 128 + 63) == EINVAL and call(d=src + 100) == EINVAL
        assert call(s=dst - 63 * 128 - 1, ss=128) == EINVAL
    assert not mem.any() and (k == 1).all() and (g == 0x3F).all()
    assert emusao.emu_launch_count() == before
