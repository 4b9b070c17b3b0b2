"""GPU tier: the exhaustive motion search (b200_me_esa_device / b200_me_esa_host) on every row of cases.ESA_CASES, and every
(fn, idx) of b200_me_cmp_batch_device in three memory layouts, bit for bit against the oracle (oracle/mecmp_oracle.c), which the CPU
tier pins to the compiled reference.  Outputs are pre-filled with a byte sentinel: what a call must not write is checked too."""
import ctypes as C
import re

import numpy as np
import pytest

import cpulibs as cl
from cases import B200_ENOSYS, ESA_CASES, ESA_INPUTS_ALL, esa_buffers, esa_expected, esa_kernel_for

pytestmark = pytest.mark.gpu
SENT = 0xA7
B200_EINVAL = -22


def on_stream(device):
    import torch
    return torch.cuda.stream(torch.cuda.ExternalStream(device.stream))


# ---------------------------------------------------------------------------------------------- exhaustive search
def _nmb(row):
    return (row["w"] // row["mb"]) * (row["h"] // row["mb"])


def _outputs(row, mv_bytes, cost_bytes):
    """(mv [nf, blocks, 2], cost [nf, blocks] uint64, both 64-entry tails still hold the sentinel)"""
    nf, nmb = row["nf"], _nmb(row)
    mv = mv_bytes[:nf * nmb * 8].view(np.int32).reshape(nf, nmb, 2)
    cost = cost_bytes[:nf * nmb * 8].view(np.uint64).reshape(nf, nmb)
    tails = bool((mv_bytes[nf * nmb * 8:] == SENT).all() and (cost_bytes[nf * nmb * 8:] == SENT).all())
    return mv, cost, tails


def esa_device(device, row, cb, rb, profile=False):
    """One b200_me_esa_device call on the row's buffers: (return code, mv, cost, tails intact, cur / ref unchanged, kernel names)"""
    import torch
    from ffmpeg_b200._lib import lib, vp
    nb = (row["nf"] * _nmb(row) + 64) * 8
    with on_stream(device):
        dc, dr = torch.from_numpy(cb).cuda(), torch.from_numpy(rb).cuda()
        dmv, dcost = (torch.full((nb,), SENT, dtype=torch.uint8, device="cuda") for _ in range(2))
        device.sync()
        names = []

        def call():
            return lib().b200_me_esa_device(device.handle, vp(dc.data_ptr() + row["cur_off"]), vp(dr.data_ptr() + row["ref_off"]),
                                            row["linesize"], row["w"], row["h"], row["frame_stride"], row["nf"], row["mb"], row["search"],
                                            vp(dmv.data_ptr()), vp(dcost.data_ptr()))
        if profile:
            from torch.profiler import ProfilerActivity
            with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
                rc = call()
                device.sync()
            names = sorted({e.key for e in prof.key_averages() if "esa" in e.key})
        else:
            rc = call()
            device.sync()
        mv, cost, tails = _outputs(row, dmv.cpu().numpy(), dcost.cpu().numpy())
        same_in = np.array_equal(dc.cpu().numpy(), cb) and np.array_equal(dr.cpu().numpy(), rb)
    return rc, mv, cost, tails, same_in, names


def _checked(row, a):
    """the macroblock rows a case compares (all, or the few the oracle has time for at 4K / 1080p)"""
    if not row["rows"]:
        return a
    bw = row["w"] // row["mb"]
    return a.reshape(a.shape[0], -1, bw, *a.shape[2:])[:, list(row["rows"])]


def _id(row):
    return f"{row['w']}x{row['h']}_mb{row['mb']}_s{row['search']}_n{row['nf']}" + ("_layout" if row["cur_off"] else "")


@pytest.mark.parametrize("row", ESA_CASES, ids=[_id(r) for r in ESA_CASES])
def test_esa_case(device, row):
    """Every input of the row: vectors and costs bit for bit against the oracle, nothing written past the outputs, inputs unchanged;
    a search without a kernel returns B200_ENOSYS and writes nothing."""
    O = cl.oracle()
    assert esa_kernel_for(row["mb"], row["search"]) == row["expect"]
    for kind in row["inputs"]:
        cb, rb, _, _ = esa_buffers(row, kind)
        rc, mv, cost, tails, same_in, _ = esa_device(device, row, cb, rb)
        assert tails and same_in, (kind, tails, same_in)
        if row["expect"] == B200_ENOSYS:
            assert rc == B200_ENOSYS, rc
            assert (mv.view(np.uint8) == SENT).all() and (cost.view(np.uint8) == SENT).all()
            continue
        assert rc == 0, rc
        emv, ecost = esa_expected(O.orc_esa_frame, row, cb, rb)
        gm, em, gc, ec = _checked(row, mv), _checked(row, emv), _checked(row, cost), _checked(row, ecost)
        bad = np.argwhere((gm != em).any(-1) | (gc != ec))
        assert bad.size == 0, (kind, len(bad), [(tuple(int(v) for v in b), gm[tuple(b)].tolist(), em[tuple(b)].tolist(),
                                                 int(gc[tuple(b)]), int(ec[tuple(b)])) for b in bad[:4]])


def _kernel(name):
    return "esa2" if "esa2_kernel" in name else "esa" if re.search(r"(?<!\w)esa_kernel<|10esa_kernelI", name) else None


@pytest.mark.parametrize("mb", [16, 8, 4])
def test_esa_boundary_kernels_agree(device, mb):
    """The searches just below and above the esa2 / esa boundary, and esa's last one, on a frame all three windows cover: the same
    vectors and costs from both kernels on every input; under torch.profiler, the kernel each one launched is the one
    cases.esa_kernel_for predicts, and the first search past the limit launches none."""
    group = [r for r in ESA_CASES if r["group"] == f"boundary{mb}"]
    assert [r["expect"] for r in group] == ["esa2", "esa", "esa"]
    for kind in ESA_INPUTS_ALL:
        cb, rb, _, _ = esa_buffers(group[0], kind)
        outs = [esa_device(device, r, cb, rb)[1:3] for r in group]
        for r, (mv, cost) in zip(group[1:], outs[1:]):
            assert np.array_equal(mv, outs[0][0]) and np.array_equal(cost, outs[0][1]), (kind, r["search"])
    enosys = next(r for r in ESA_CASES if r["mb"] == mb and r["expect"] == B200_ENOSYS and r["w"] == group[0]["w"])
    cb, rb, _, _ = esa_buffers(group[0], "random")
    for r in group + [enosys]:
        rc, _, _, _, _, names = esa_device(device, r, cb, rb, profile=True)
        kinds = {_kernel(n) for n in names} - {None}
        if r["expect"] == B200_ENOSYS:
            assert rc == B200_ENOSYS and not kinds, (rc, names)
        else:
            assert rc == 0 and kinds == {r["expect"]}, (r["search"], names)
            assert any(f"<{mb}" in n or f"ILi{mb}E" in n for n in names), names


def test_me_esa_host_slot_reuse(device):
    """b200_me_esa_host with a frame_stride that makes each chunk of its 96 MB staging two frames: 7 frames are 4 chunks over the three
    pipeline slots, so slot 0 is used twice.  Against the oracle and the device entry; a search past the limit returns B200_ENOSYS
    through this entry too and writes nothing."""
    from ffmpeg_b200 import me_cmp
    from ffmpeg_b200._lib import lib, vp
    row = dict(w=64, h=48, linesize=64, frame_stride=17 << 20, cur_off=0, ref_off=0, nf=7, mb=16, search=16, rows=None)
    nmb = _nmb(row)
    per_frame = 2 * row["frame_stride"] + ((nmb * 16 + 255) & ~255)
    assert (96 << 20) // per_frame == 2                            # csrc/mecmp.cu b200_me_esa_host: frames per chunk
    cb, rb, _, _ = esa_buffers(row, "shifted")
    mvb, costb = (np.full((row["nf"] * nmb + 64) * 8, SENT, np.uint8) for _ in range(2))
    me_cmp.me_esa_host(device, cb, rb, row["linesize"], row["w"], row["h"], row["frame_stride"], row["nf"], row["mb"], row["search"],
                       mvb, costb)
    mv, cost, tails = _outputs(row, mvb, costb)
    assert tails
    emv, ecost = esa_expected(cl.oracle().orc_esa_frame, row, cb, rb)
    assert np.array_equal(mv, emv) and np.array_equal(cost, ecost)
    rc, dmv, dcost, _, _, _ = esa_device(device, row, cb, rb)
    assert rc == 0 and np.array_equal(dmv, mv) and np.array_equal(dcost, cost)
    mvb[:], costb[:] = SENT, SENT
    rc = lib().b200_me_esa_host(device.handle, vp(cb.ctypes.data), vp(rb.ctypes.data), row["linesize"], row["w"], row["h"],
                                row["frame_stride"], row["nf"], 16, 217, vp(mvb.ctypes.data), vp(costb.ctypes.data))
    assert rc == B200_ENOSYS and (mvb == SENT).all() and (costb == SENT).all(), rc


# ---------------------------------------------------------------------------------------------- block compare
# every (fn, idx) b200_me_cmp_batch_device accepts, with the heights it is run at
_H_PLAIN, _H_HAD, _H_GRAD = (1, 2, 7, 8, 15, 16), (4, 8, 16), (1, 2, 7, 8, 16)
CMP_FNS = {0: [(i, _H_PLAIN) for i in (0, 1)], 1: [(i, _H_PLAIN) for i in (0, 1, 2)], 2: [(i, _H_PLAIN) for i in range(8)],
           3: [(i, _H_HAD) for i in (0, 1, 4, 5)]}
for _fn in (4, 5):
    CMP_FNS[_fn] = [(i, _H_GRAD + ((32,) if i & 1 else ())) for i in (0, 1, 4, 5)]
for _fn in (6, 7):
    CMP_FNS[_fn] = [(0, _H_GRAD), (1, _H_GRAD + (32,))]
for _fn in (8, 9, 10):
    CMP_FNS[_fn] = [(i, _H_HAD) for i in (0, 1)]
CMP_NAMES = {0: "sad", 1: "sse", 2: "pix_abs", 3: "hadamard8", 4: "vsad", 5: "vsse", 6: "nsse", 7: "median_sad", 8: "dct_sad",
             9: "dct_max", 10: "dct264_sad"}
CMP_INPUTS = ("random", "near", "extremes", "flat")
# (stride, byte offset of frame1 and frame2 in their buffers); C: rows go up in memory, offsets point at the bottom rows
CMP_LAYOUTS = {"A": (256, 0, 0), "B": (203, 1, 3), "C": (-256, 0, 0)}
CMP_N, CMP_ROWS = 4099, 96


def cmp_case(layout, kind):
    """(buffer 1, buffer 2, frame1 offset, frame2 offset, stride, off1, off2): CMP_N block pairs of one input kind in one layout.  Blocks
    leave room for 33 rows and 17 columns (x2 / y2 / xy2 read one more of each)."""
    stride, b1, b2 = CMP_LAYOUTS[layout]
    s = abs(stride)
    rng = np.random.default_rng(100 * ord(layout) + CMP_INPUTS.index(kind))
    shape = CMP_ROWS * s + 64
    if kind == "random":
        f1, f2 = rng.integers(0, 256, shape, dtype=np.uint8), rng.integers(0, 256, shape, dtype=np.uint8)
    elif kind == "near":
        f1 = rng.integers(0, 256, shape, dtype=np.uint8)
        f2 = (f1.astype(np.int16) + rng.integers(-3, 4, shape)).clip(0, 255).astype(np.uint8)
    elif kind == "extremes":
        f1, f2 = (rng.integers(0, 2, shape) * 255).astype(np.uint8), (rng.integers(0, 2, shape) * 255).astype(np.uint8)
    else:
        f1, f2 = np.full(shape, 200, np.uint8), np.full(shape, 13, np.uint8)
    buf1, buf2 = (np.concatenate([rng.integers(0, 256, b, dtype=np.uint8), f]) for b, f in ((b1, f1), (b2, f2)))
    pos = []
    for _ in range(2):
        y, x = rng.integers(0, CMP_ROWS - 33, CMP_N), rng.integers(0, s - 17, CMP_N)
        pos.append(((CMP_ROWS - 1 - y) if stride < 0 else y) * s + x)
    off1, off2 = (p.astype(np.int64) for p in pos)
    if kind == "near":
        off2 = off1.copy()
    return buf1, buf2, b1, b2, stride, off1, off2


def cmp_expected(fn, idx, h, buf1, buf2, b1, b2, stride, off1, off2):
    out = np.zeros(len(off1), np.int32)
    cl.oracle().orc_me_cmp_batch(fn, idx, buf1.ctypes.data + b1, buf2.ctypes.data + b2, stride, h, off1.ctypes.data, off2.ctypes.data,
                                 len(off1), out.ctypes.data)
    return out


@pytest.mark.parametrize("layout", list(CMP_LAYOUTS))
@pytest.mark.parametrize("fn", list(CMP_FNS), ids=[CMP_NAMES[f] for f in CMP_FNS])
def test_me_cmp_batch_device(device, fn, layout):
    """Every index and height of one family, for 1, 9 and 4099 block pairs of each input: every output against the oracle, and the
    64 entries past n keep their sentinel."""
    import torch
    from ffmpeg_b200 import me_cmp
    cl.oracle().orc_me_cmp_set_dct_algo(0)
    me_cmp.me_cmp_set_dct_algo(me_cmp.FF_DCT_AUTO)
    for kind in CMP_INPUTS:
        buf1, buf2, b1, b2, stride, off1, off2 = cmp_case(layout, kind)
        with on_stream(device):
            d1, d2 = torch.from_numpy(buf1).cuda(), torch.from_numpy(buf2).cuda()
            o1, o2 = torch.from_numpy(off1).cuda(), torch.from_numpy(off2).cuda()
            for idx, hs in CMP_FNS[fn]:
                for h in hs:
                    exp = cmp_expected(fn, idx, h, buf1, buf2, b1, b2, stride, off1, off2)
                    for n in (1, 9, CMP_N):
                        out = torch.full((n + 64,), SENT * 0x01010101 - (1 << 32), dtype=torch.int32, device="cuda")
                        me_cmp.me_cmp_batch_device(device, fn, idx, d1.data_ptr() + b1, d2.data_ptr() + b2, stride, h, o1, o2, n, out)
                        device.sync()
                        got = out.cpu().numpy()
                        bad = np.flatnonzero(got[:n] != exp[:n])
                        assert bad.size == 0, (kind, idx, h, n, len(bad), [(int(i), int(got[i]), int(exp[i])) for i in bad[:4]])
                        assert (got[n:].view(np.uint8) == SENT).all(), (kind, idx, h, n)


def test_me_cmp_batch_device_refuses_large_blocks(device):
    """vsad / vsse / nsse / median_sad take at most 256 pixels (w * h): larger blocks return B200_EINVAL and write nothing."""
    import torch
    from ffmpeg_b200._lib import lib, vp
    buf1, buf2, b1, b2, stride, off1, off2 = cmp_case("A", "random")
    with on_stream(device):
        d1, d2 = torch.from_numpy(buf1).cuda(), torch.from_numpy(buf2).cuda()
        o1, o2 = torch.from_numpy(off1).cuda(), torch.from_numpy(off2).cuda()
        for fn in (4, 5, 6, 7):
            for idx, hs in CMP_FNS[fn]:
                h = 17 if not idx & 1 else 33
                out = torch.full((80,), -1, dtype=torch.int32, device="cuda")
                rc = lib().b200_me_cmp_batch_device(device.handle, fn, idx, vp(d1.data_ptr()), vp(d2.data_ptr()), stride, h,
                                                    vp(o1.data_ptr()), vp(o2.data_ptr()), 16, vp(out.data_ptr()))
                device.sync()
                assert rc == B200_EINVAL and (out.cpu().numpy() == -1).all(), (fn, idx, h, rc)


def test_nsse_weight(device):
    """b200_me_cmp_set_nsse_weight (the drop-in's stand-in for avctx->nsse_weight) at several weights: the batched entry and the
    function table against the oracle at the same weight.  The weight is process-wide: 8, the NULL-context weight, is restored."""
    import torch
    from ffmpeg_b200 import me_cmp
    O = cl.oracle()
    c = me_cmp.ff_me_cmp_init()
    try:
        for kind in ("random", "near"):
            buf1, buf2, b1, b2, stride, off1, off2 = cmp_case("B", kind)
            with on_stream(device):
                d1, d2 = torch.from_numpy(buf1).cuda(), torch.from_numpy(buf2).cuda()
                o1, o2 = torch.from_numpy(off1).cuda(), torch.from_numpy(off2).cuda()
                out = torch.zeros(CMP_N, dtype=torch.int32, device="cuda")
                for wgt in (0, 1, 8, 37, -5):
                    me_cmp.me_cmp_set_nsse_weight(wgt)
                    O.orc_me_cmp_set_nsse_weight(wgt)
                    for idx, hs in CMP_FNS[6]:
                        for h in hs:
                            exp = cmp_expected(6, idx, h, buf1, buf2, b1, b2, stride, off1, off2)
                            me_cmp.me_cmp_batch_device(device, 6, idx, d1.data_ptr() + b1, d2.data_ptr() + b2, stride, h, o1, o2, CMP_N, out)
                            device.sync()
                            assert np.array_equal(out.cpu().numpy(), exp), (kind, wgt, idx, h)
                            for i in range(0, CMP_N, 400):
                                p1 = C.cast(buf1.ctypes.data + b1 + int(off1[i]), cl.u8p)
                                p2 = C.cast(buf2.ctypes.data + b2 + int(off2[i]), cl.u8p)
                                assert c.nsse[idx](None, p1, p2, stride, h) == exp[i], (kind, wgt, idx, h, i)
    finally:
        me_cmp.me_cmp_set_nsse_weight(8)
        O.orc_me_cmp_set_nsse_weight(8)
