"""CPU tier for VP9 intra reconstruction (VP9DSPContext's intra_pred members and b200_vp9_intra_recon_frame_device,
ffmpeg_b200/csrc/vp9intra.cu): the checker (oracle/vp9intra_oracle.c) against the compiled reference (oracle/_ref/libffref_vp9intra.so)
on all 60 members at every depth and on whole generated frames (every chroma format, odd sizes, tight line sizes that take the decoder's
emulated-edge path, tile columns, lossless, skip, intra blocks among inter samples); the fixture hashes; the fixture frames telling the
decode order apart from an order without dependencies; the layouts; and vp9intra.cu itself, host code included, on the stand-in CUDA
runtime of tests/cuda_emu (fixture frames with sentinels, every member at every depth with everything outside its footprint poisoned,
invalid ops, the init's table, refusals)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cpulibs as cl
import vp9intralib as vi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "cuda_emu")
EINVAL, ENOSYS = -22, -38


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------- the checker against the reference
@pytest.mark.parametrize("depth", vi.DEPTHS)
@pytest.mark.parametrize("edges", ("random", "low", "high"))
def test_checker_members_match_reference(depth, edges):
    """all 60 members, three calls each, on random edges and on edges at both clip bounds (TM's clip, the averages' carries)"""
    calls = list(vi.member_calls(10 * depth + len(edges), depth, edges=edges))
    ours = [vi.run_member(vi.orc_member(depth, c[0], c[1]), depth, c) for c in calls]
    with vi.RefCheck() as rc:
        assert rc.same(ours, lambda: [vi.run_member(vi.ref_member(depth, c[0], c[1]), depth, c) for c in calls])


FRAMES = {
    "8-420-intra": (8, "420", 328, 200, {}),
    "10-422-intra-tiles": (10, "422", 400, 136, {"tiles": 3}),
    "12-440-inter": (12, "440", 264, 150, {"kind": "inter", "p_intra": 0.5}),
    "8-444-lossless": (8, "444", 121, 97, {"lossless": True}),
    "10-420-4x4-odd": (10, "420", 203, 121, {"sizes": "4x4"}),
    "12-444-skip": (12, "444", 140, 70, {"p_skip": 0.7}),
    "8-422-inter-4x4": (8, "422", 190, 66, {"kind": "inter", "sizes": "4x4", "p_intra": 0.5}),
    "10-440-lossless-tiles": (10, "440", 520, 40, {"lossless": True, "tiles": 4}),
}


@pytest.mark.parametrize("name", list(FRAMES))
@pytest.mark.parametrize("tight", (False, True), ids=("wide", "tight"))
def test_checker_frames_match_reference(name, tight):
    """whole frames, the reference's ff_vp9_intra_recon_* block by block: with line sizes of the 8-aligned width (the decoder's
    emulated-edge buffers for every block that passes it, with their copy-back) and with wide ones; the same samples either way"""
    depth, fmt, w, h, kw = FRAMES[name]
    f = vi.Frame(300 + len(name) + depth, depth, fmt, w, h, **kw)
    assert len(f.ops) > 0
    ours = f.area(vi.orc_frame(f))
    assert not same(ours, f.area(f.planes))
    with vi.RefCheck() as rc:
        assert rc.same(ours, lambda: vi.ref_frame(f, tight=tight))


@pytest.mark.parametrize("name", vi.FIXTURE_NAMES)
def test_fixture_hashes(name):
    """the checker gives the reference's hash on every fixture frame (sentinels included)"""
    f = vi.frame_case(name)
    assert vi.digest(vi.orc_frame(f)) == vi.fixture_hashes()[name]


@pytest.mark.parametrize("name", vi.FIXTURE_NAMES)
def test_fixtures_need_the_dependencies(name):
    """every fixture frame comes out differently when each op reads the planes as they were before the call: a missing wait shows"""
    f = vi.frame_case(name)
    assert not same(vi.orc_frame(f, order=1), vi.orc_frame(f))


def test_layouts():
    """INTRA_DTYPE = Vp9IntraOp = B200Vp9IntraOp (32 bytes, static_assert in the header); intra_pred is the first member of the context
    mirror (the reference harness asserts the same of VP9DSPContext)"""
    from ffmpeg_b200 import vp9dsp
    from ffmpeg_b200._lib import VP9DSPContext, Vp9IntraOp
    assert C.sizeof(Vp9IntraOp) == vp9dsp.INTRA_DTYPE.itemsize == 32
    for name in ("coef_off", "x", "y", "eob", "plane", "tx", "mode", "flags"):
        assert getattr(Vp9IntraOp, name).offset == vp9dsp.INTRA_DTYPE.fields[name][1], name
    assert VP9DSPContext.intra_pred.offset == 0 and VP9DSPContext.itxfm_add.offset == 60 * 8
    hdr = open(os.path.join(ROOT, "include", "b200dsp.h")).read()
    assert 'static_assert(sizeof(B200Vp9IntraOp) == 32, "B200Vp9IntraOp is 32 bytes");' in hdr
    assert (vp9dsp.INTRA_HAVE_LEFT, vp9dsp.INTRA_HAVE_RIGHT, vp9dsp.INTRA_LOSSLESS) == (1, 2, 4)
    if vi.have_ref():
        for tx in range(4):
            for mode in range(15):                           # at 12 bit, all but TM and DC_127 / 128 / 129 are the 10-bit functions
                assert vi.ref().ffref_vp9_intra_shared10(12, tx, mode) == (mode not in (9, 12, 13, 14))


# ---------------------------------------------------------------- vp9intra.cu on the stand-in runtime
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
"""


def emu_source(text_fn=None):
    src = open(os.path.join(ROOT, "ffmpeg_b200", "csrc", "vp9intra.cu")).read()
    if text_fn:
        src = text_fn(src)
    a, b = src.index("// ---- inter-warp progress\n"), src.index("// ---- end of inter-warp progress")
    return "#include <chrono>\n" + src[:a] + PROGRESS_EMU + src[b:]


def build_emu(name, text_fn=None):
    """lib<name>.so: vp9intra.cu (after text_fn, if given) with its host code, vp9mc.cu (b200_vp9_dsp_init) and vp9itxfm.cu, compiled with
    g++ against tests/cuda_emu/fake/cuda_runtime.h.  The frame kernel's progress helpers (PTX) become host atomics and a real clock, its
    static shared arrays statics (blocks run one at a time), and every thread of a block is an OS thread, so the warps of a block wait
    on one another for real."""
    from test_cuda_emu import rewrite_launches
    gen = os.path.join(EMU, "_gen")
    os.makedirs(gen, exist_ok=True)
    cs = os.path.join(ROOT, "ffmpeg_b200", "csrc")
    srcs = []
    for f in ("vp9intra.cu", "vp9mc.cu", "tx_pfa.cu"):           # tx_pfa.cu: fake_device.cpp links it
        src = emu_source(text_fn) if f == "vp9intra.cu" else open(os.path.join(cs, f)).read()
        t = rewrite_launches(src)
        t = t.replace("extern __shared__ float2 pfa_z[];", "float2 *pfa_z = (float2 *)emu_smem;")
        if f == "vp9intra.cu":
            assert t.count("emu_cfg_launch(0, [&] { vp9_intra_kernel<") == 2 and t.count("emu_cfg_launch(0, [&] { vp9_intra_member_kernel<") == 2
            assert "asm" not in t
            t = t.replace("emu_cfg_launch(0, [&] { vp9_intra_kernel<", "emu_cfg_launch(2, [&] { vp9_intra_kernel<")
            t = t.replace("emu_cfg_launch(0, [&] { vp9_intra_member_kernel<", "emu_cfg_launch(2, [&] { vp9_intra_member_kernel<")
            t = t.replace("__shared__", "static")
            t = t.replace("__syncwarp();", "emu_bwarp->bar->arrive_and_wait();")
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
    L.b200_vp9_dsp_init_intrapred.argtypes = [C.c_void_p, C.c_int]
    L.b200_vp9_intra_recon_frame_device.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int64,
                                                                                   C.c_void_p, C.c_void_p]
    L.b200_vp9_intra_timeouts.argtypes = [C.c_void_p, C.c_void_p]
    L.emu_launch_count.restype = C.c_uint64
    return L


@pytest.fixture(scope="module")
def emuintra():
    return build_emu("emuvp9intra")


def emu_frame(L, f, ops=None):
    """the frame entry on copies of the planes (sentinels included); coef in a 16-byte aligned buffer"""
    out = [p.copy() for p in f.planes]
    arr = (C.c_void_p * 3)(*f.ptrs(out))
    ops = np.ascontiguousarray(f.ops if ops is None else ops)
    raw = f.coef.view(np.uint8)
    buf = np.zeros(raw.size + 64, np.uint8)
    start = -buf.ctypes.data % 16
    buf[start:start + raw.size] = raw
    ls_y, ls_uv = f.strides()
    assert L.b200_vp9_intra_recon_frame_device(None, f.depth, f.ss_h, f.ss_v, f.width, f.height, arr, ls_y, ls_uv, len(ops), ops.ctypes.data,
                                               buf.ctypes.data + start) == 0
    assert np.array_equal(buf[start:start + raw.size], raw)
    return out


def emu_timeouts(L):
    n = C.c_int64(-1)
    assert L.b200_vp9_intra_timeouts(None, C.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("name", vi.FIXTURE_NAMES)
def test_emu_frame_vs_checker_and_fixture(emuintra, name):
    """the fixture frame through the library's entry: equal to the checker over the whole arrays (the sentinels around every plane
    unchanged) and to the reference's hash; no wait ran out"""
    f = vi.frame_case(name)
    got = emu_frame(emuintra, f)
    assert same(got, vi.orc_frame(f))
    assert vi.digest(got) == vi.fixture_hashes()[name]
    assert emu_timeouts(emuintra) == 0


@pytest.mark.parametrize("depth", vi.DEPTHS)
def test_emu_extreme_coefficients(emuintra, depth):
    """a frame whose coefficients are the storage type's extremes and full-range values (vp9itxfmlib's "extremes" class): the transform
    passes' truncation and wrapping are the reference's (the checker's residual is vp9itxfm_oracle.c, compared with the reference on
    the same class)"""
    f = extreme_frame(depth)
    assert same(emu_frame(emuintra, f), vi.orc_frame(f))


def extreme_frame(depth):
    import vp9itxfmlib as vt
    f = vi.Frame(40 + depth, depth, "444", 136, 72, p_skip=0.0, lossless=depth == 12)
    rng = np.random.default_rng(depth)
    for k in range(len(f.ops)):
        t = 4 if f.lossless else int(f.ops["tx"][k])
        b, eob = vt.coefs(rng, depth, t, "extremes")
        f.ops["eob"][k] = max(eob, 2) if k % 3 else 1
        f.coef[f.ops["coef_off"][k]:f.ops["coef_off"][k] + b.size] = b.ravel()
    return f


@pytest.mark.parametrize("seed", range(4))
def test_emu_blocks_past_the_right_edge(emuintra, seed):
    """narrow frames (9 columns of 8x8 blocks, so the second superblock column is one 8x8 wide) whose 16x16 and 32x32 transform blocks
    pass the plane's right edge: the top row is replicated from the last sample inside the plane, nothing past it is read or written"""
    f = vi.Frame(60 + seed, 8 + 2 * (seed & 1), "420", 72, 136)
    o = f.ops
    assert ((4 << o["tx"].astype(int)) > np.array(f.W)[o["plane"]] - o["x"]).any()
    assert same(emu_frame(emuintra, f), vi.orc_frame(f))


def test_emu_invalid_ops(emuintra):
    """ops with a plane, tx or mode out of range, unaligned x / y / coef_off, LOSSLESS with tx > 0, or outside the plane write nothing
    and hold up no later op: the frame with them mixed in equals the frame without them"""
    f = vi.frame_case("420-8-intra")
    rng = np.random.default_rng(3)
    bad = np.zeros(9, f.ops.dtype)
    bad["eob"] = 5
    bad["plane"][0], bad["tx"][1], bad["mode"][2] = 3, 4, 10
    bad["x"][3], bad["y"][4], bad["coef_off"][5] = 2, 6, 8
    bad["flags"][6], bad["tx"][6] = 4, 1
    bad["x"][7], bad["y"][8] = f.W[0], f.H[0] + 4
    mixed = np.insert(f.ops, rng.integers(0, len(f.ops), len(bad)), bad)
    want = vi.orc_frame(f)
    assert same(emu_frame(emuintra, f, mixed), want)
    g = vi.frame_case("420-8-intra")
    g.ops = mixed
    assert same(vi.orc_frame(g), want)
    assert emu_timeouts(emuintra) == 0


@pytest.mark.parametrize("depth", vi.DEPTHS)
def test_emu_every_member(emuintra, depth):
    """every member through host pointers against the checker, on edges where every sample the reference does not read is poisoned:
    the member reads nothing outside its footprint, and writes exactly its block (sentinels around it stay)"""
    from ffmpeg_b200._lib import VP9DSPContext
    from ffmpeg_b200.vp9dsp import VP9_INTRA_FUNC
    ctx = VP9DSPContext()
    assert emuintra.b200_vp9_dsp_init_intrapred(C.byref(ctx), depth) == 0
    st = vi.sdtype(depth)
    probe = vi.ref_member if vi.have_ref() else vi.orc_member
    for tx, mode, left, top, dst0 in vi.member_calls(50 + depth, depth, per=2):
        n = 4 << tx
        want = vi.run_member(vi.orc_member(depth, tx, mode), depth, (tx, mode, left, top, dst0))
        for poison in (0, (1 << depth) - 1):
            # the footprint: samples whose change changes the checker's result are kept, the rest poisoned; a wider buffer around both
            lb = np.full(n + 16, poison, st)
            tb = np.full(2 * n + 1 + 16, poison, st)
            lb[8:8 + n], tb[8:8 + 2 * n + 1] = left, top
            keep_l, keep_t = footprint(depth, tx, mode, probe)
            lb[8:8 + n][~keep_l] = poison
            tb[8:8 + 2 * n + 1][~keep_t] = poison
            d = np.full((n + 8, n + 8), 7, st)
            d[4:4 + n, 4:4 + n] = dst0
            VP9_INTRA_FUNC(ctx.intra_pred[tx][mode])(d.ctypes.data + 4 * d.strides[0] + 4 * d.itemsize, d.strides[0],
                                                     lb.ctypes.data + 8 * lb.itemsize, tb.ctypes.data + 9 * tb.itemsize)
            assert np.array_equal(d[4:4 + n, 4:4 + n], vi.run_member(vi.orc_member(depth, tx, mode), depth,
                                                                     (tx, mode, lb[8:8 + n], tb[8:8 + 2 * n + 1], dst0))), (depth, tx, mode)
            inner = d[4:4 + n, 4:4 + n].copy()
            d[4:4 + n, 4:4 + n] = 7
            assert (d == 7).all(), (depth, tx, mode)
            if keep_l.all() and keep_t[1:n + 1].all():
                assert np.array_equal(inner, want)


_fp = {}


def footprint(depth, tx, mode, member):
    """which left[] / top[-1 ..] samples member `mode` reads: those whose change (to 0 and to the maximum) changes its output"""
    key = (depth, tx, mode, member)
    if key not in _fp:
        n, st, mx = 4 << tx, vi.sdtype(depth), (1 << depth) - 1
        rng = np.random.default_rng(tx * 15 + mode)
        base_l, base_t = rng.integers(1, mx, n).astype(st), rng.integers(1, mx, 2 * n + 1).astype(st)
        d0 = np.zeros((n, n), st)
        ref = vi.run_member(member(depth, tx, mode), depth, (tx, mode, base_l, base_t, d0))
        keep_l, keep_t = np.zeros(n, bool), np.zeros(2 * n + 1, bool)
        for arr, keep, is_left in ((base_l, keep_l, True), (base_t, keep_t, False)):
            for k in range(arr.size):
                for v in (0, mx):
                    a = arr.copy()
                    a[k] = v
                    args = (tx, mode, a, base_t, d0) if is_left else (tx, mode, base_l, a, d0)
                    if not np.array_equal(vi.run_member(member(depth, tx, mode), depth, args), ref):
                        keep[k] = True
        _fp[key] = (keep_l, keep_t)
    return _fp[key]


def table_words(ctx):
    return np.frombuffer(C.string_at(C.addressof(ctx), C.sizeof(ctx)), np.uint64)


def test_emu_init_sets_exactly_the_table(emuintra):
    """on top of b200_vp9_dsp_init's context the init sets the 60 intra_pred words (0..59) and nothing else; 60 distinct functions per
    depth; at 12 bit all but TM and DC_127 / 128 / 129 are the 10-bit functions"""
    from ffmpeg_b200._lib import VP9DSPContext
    words = {}
    for depth in vi.DEPTHS:
        ctx = VP9DSPContext()
        assert emuintra.b200_vp9_dsp_init(C.byref(ctx), depth) == 0
        w0 = table_words(ctx).copy()
        assert emuintra.b200_vp9_dsp_init_intrapred(C.byref(ctx), depth) == 0
        w1 = table_words(ctx)
        assert list(np.nonzero(w0 != w1)[0]) == list(range(60))
        assert len(set(w1[:60])) == 60
        words[depth] = w1[:60].reshape(4, 15)
    shared = words[12] == words[10]
    assert (shared[:, [9, 12, 13, 14]] == False).all() and shared[:, [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 11]].all()  # noqa: E712
    assert not (words[8] == words[10]).any()


# ---------------------------------------------------------------- refusals (argument checks come before the device)
@pytest.fixture(scope="module")
def prodlib():
    import ffmpeg_b200
    return ffmpeg_b200.lib()


def test_init_refusals(prodlib, emuintra):
    from ffmpeg_b200._lib import VP9DSPContext
    for L in (prodlib, emuintra):
        ctx = VP9DSPContext()
        for depth in (0, 7, 9, 11, 13, 14, 16):
            assert L.b200_vp9_dsp_init_intrapred(C.byref(ctx), depth) == ENOSYS, depth
        assert L.b200_vp9_dsp_init_intrapred(None, 8) == EINVAL
        assert not table_words(ctx).any()


def test_frame_refusals(prodlib, emuintra):
    """every B200_EINVAL case launches nothing (the buffers stay zero, the stand-in runtime's launch count does not move); nops == 0
    returns 0 without a launch"""
    b = np.zeros(1 << 16, np.uint8)
    p = b.ctypes.data + (-b.ctypes.data % 64)
    before = emuintra.emu_launch_count()
    for L in (prodlib, emuintra):
        def call(depth=8, ss_h=1, ss_v=1, w=64, h=64, planes=(p, p + 8192, p + 12288), ls_y=64, ls_uv=32, nops=1, ops=p + 16384,
                 coef=p + 32768):
            arr = (C.c_void_p * 3)(*planes) if planes is not None else None
            return L.b200_vp9_intra_recon_frame_device(None, depth, ss_h, ss_v, w, h, arr, ls_y, ls_uv, nops, ops, coef)
        for depth in (0, 7, 9, 11, 13, 16):
            assert call(depth=depth) == EINVAL, depth
        assert call(ss_h=2) == EINVAL and call(ss_v=-1) == EINVAL
        assert call(w=0) == EINVAL and call(h=0) == EINVAL and call(w=-5) == EINVAL and call(w=65537) == EINVAL
        assert call(planes=None) == EINVAL and call(planes=(p, None, p)) == EINVAL
        assert call(nops=-1) == EINVAL and call(nops=(1 << 30) + 1) == EINVAL
        assert call(ops=None) == EINVAL and call(coef=None) == EINVAL and call(ops=p + 16388) == EINVAL and call(coef=p + 32776) == EINVAL
        assert call(ls_y=63) == EINVAL and call(ls_uv=31) == EINVAL and call(w=65, ls_y=64) == EINVAL and call(ss_h=0, ls_uv=32) == EINVAL
        assert call(depth=10, ls_y=128, ls_uv=63) == EINVAL and call(depth=10, ls_y=129, ls_uv=64) == EINVAL
        assert call(depth=10, ls_y=128, ls_uv=64, planes=(p + 1, p + 8192, p + 12288)) == EINVAL
        assert call(depth=12, ls_y=128, ls_uv=64, planes=(p, p + 8192, p + 12289)) == EINVAL
        assert call(nops=0, ops=None, coef=None) == 0
        assert L.b200_vp9_intra_timeouts(None, None) == EINVAL
    assert not b.any()
    assert emuintra.emu_launch_count() == before
