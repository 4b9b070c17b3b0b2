"""GPU tier: every route of the 8-bit simple IDCT, the inverse quantisers and the 10 / 12 bit and ProRes IDCTs, bit for bit against
the checker (oracle/), at the geometries, strides and coefficients the dispatchers branch on.

Each case is built so that the dispatcher must take a known route, named first in the case id.  test_route_launches checks that
every case shape launches the route's kernel with the grid and block the dispatcher must pick (recorded with torch.profiler in a
child process, see record_routes).  The routes:
  tiled    idct_mb420_kernel<KIND> (b200_idct_mb420_device): planes, line sizes and frame strides 16-byte (luma) / 8-byte (chroma)
           aligned, line sizes > 0, mb_h <= 65535 (csrc/idct.cu:644-648).  Segments of 8 macroblocks per CTA: 3, 4, 5 or 6, the width
           wasting the fewest idle segments, the wider on a tie (idct.cu:649-655; mirrored by test_idct_routes.mb420_segs).  Six
           segments need 55,296 B of dynamic shared memory, above the 48 KiB default (the cudaFuncSetAttribute opt-in, :656).  More
           than 65,535 frames go out in launches of at most 65,535 frames, each with its planes moved on by f0 frames (:657-664).
  warp     idct8x8_kernel<KIND, true>, the fallback of b200_idct_mb420_device when any condition of `tiled` fails (:703-705): luma
           line size = 8 mod 16, an odd chroma line size, a plane pointer + 1, bottom-up planes (negative line sizes), mb_h 65,536.
  tpb      idct_tpb_kernel<KIND> (b200_idct_batch_device, :339-399, 708-710): one thread per block, 128 per CTA.  Destinations
           dest + dest_off[i], line size line_size[i] (an array) or the uniform one; 8-byte row stores when the row pointer and
           the line size are both 8-byte aligned, bytes otherwise (:363).  Kind 0 works in place and writes back only the CTA's
           own nblocks - b0 blocks.  Blocks that are not 16-byte aligned are refused (:761).
  fused    idct_mb420_kernel<KIND, V> (b200_mpv_unquant_idct_mb420_device, :422-472, 671-693): the inverse quantiser fused in
           front of the tiled kernel, same CTA width choice.  Refused: unaligned planes or line sizes <= 0, nframes > 65535, a
           permutated[] that is not a permutation (:674-679, 731-737).
  unquant  mpv_unquant_kernel<V> (b200_mpv_unquantize_batch_device, csrc/unquant.cu:46-105, 110-145): one warp per block, the
           grid capped at sm_count * 16 * 8 CTAs of 4 warps, so that past 4 * 16,896 blocks (H100) every warp walks more than one
           block; blocks need only be 4-byte aligned (:117).
  hbd      idct_hbd_kernel<DEPTH, KIND> (b200_idct_hbd_batch_device, csrc/idct_hbd.cu:75-150, 249-266), depth 9 through its alias
           to 10: 16-byte row loads / stores when the row pointer and the line size are 16-byte aligned (:111), samples otherwise.
  prores   prores_idct_put_kernel<VARIANT> (b200_prores_idct_put_batch_device, idct_hbd.cu:155-180, 320-333): coefficient * qmat
           wrapped to int16, clipped to [4, 2^bits - 5].

Coefficients: every class of test_idct_routes.CLASSES (the six of tests/cases.py and dcrows, zero, saturate, maxabs) mixed in
every call.  Each destination buffer holds a sentinel in line-size padding and 256 bytes before and after what the call may write,
and the whole buffer must equal the checker's (which writes only the blocks); the coefficients of the put / add routes and
kind-0 blocks past nblocks must come back unchanged, and a refused call changes nothing and launches nothing."""
import json
import os
import tempfile

import numpy as np
import pytest

import cpulibs as cl
from test_idct_routes import (H263, LS8, LS16, MB420_WIDTHS, extreme_configs, extreme_unquant_case, footprint,
                              mb420_height, mb420_segs, mixed_blocks, orc_hbd, orc_idct8, orc_prores, private_rows, prores_qmat,
                              width_id)

pytestmark = pytest.mark.gpu

SENT = 0xA5
HEAD = TAIL = 256
KIND_NAMES = {0: "idct", 1: "put", 2: "add"}


def on_stream(device):
    import torch
    return torch.cuda.stream(torch.cuda.ExternalStream(device.stream))


def diff_report(got, exp, mask):
    bad = got != exp
    return f"{int((bad & mask).sum())} bytes differ inside what the call may write, {int((bad & ~mask).sum())} outside"


def launch_count():
    import ffmpeg_b200 as fb
    return fb.launch_count()


# ---------------------------------------------------------------------------------------------- 4:2:0 macroblock pictures
class Pics:
    """The three planes of nf frames in flat byte buffers: random pixels in the picture, SENT in the line-size padding and the
    HEAD / TAIL bytes around it.  Bottom-up planes start at their last row (negative line sizes)."""

    def __init__(self, mb_w, mb_h, nf, seed, pad=(32, 16, 16), bottom_up=False, shift=(0, 0, 0)):
        rng = np.random.default_rng(seed)
        self.mb_w, self.mb_h, self.nf = mb_w, mb_h, nf
        self.W, self.H = [16 * mb_w, 8 * mb_w, 8 * mb_w], [16 * mb_h, 8 * mb_h, 8 * mb_h]
        self.ls, self.fs, self.org, self.buf, self.mask = [], [], [], [], []
        for p in range(3):
            a = self.W[p] + pad[p]
            ls = -a if bottom_up else a
            org = HEAD + shift[p] + (self.H[p] - 1) * a * bottom_up
            buf = np.full(HEAD + shift[p] + nf * self.H[p] * a + TAIL, SENT, np.uint8)
            f = np.arange(nf, dtype=np.int64)[:, None, None] * (self.H[p] * a)
            r = np.arange(self.H[p], dtype=np.int64)[None, :, None] * ls
            c = np.arange(self.W[p], dtype=np.int64)[None, None, :]
            pos = (org + f + r + c).ravel()
            buf[pos] = rng.integers(0, 256, pos.size, dtype=np.uint8)
            mask = np.zeros(buf.size, bool)
            mask[pos] = True
            self.ls.append(ls); self.fs.append(self.H[p] * a); self.org.append(org); self.buf.append(buf); self.mask.append(mask)

    def block_offsets(self):
        """per plane: (indices of the stream's blocks in that plane, their byte offsets in the plane's buffer)"""
        per = self.mb_w * self.mb_h * 6
        b = np.arange(per * self.nf, dtype=np.int64)
        f, r = b // per, b % per
        mb, k = r // 6, r % 6
        mby, mbx = mb // self.mb_w, mb % self.mb_w
        out = []
        for p in range(3):
            sel = (k < 4) if p == 0 else (k == 3 + p)
            if p == 0:
                off = self.org[0] + f * self.fs[0] + (mby * 16 + (k >> 1) * 8) * self.ls[0] + mbx * 16 + (k & 1) * 8
            else:
                off = self.org[p] + f * self.fs[p] + mby * 8 * self.ls[p] + mbx * 8
            out.append((np.nonzero(sel)[0], off[sel]))
        return out

    def oracle(self, kind, blocks, live=None):
        """the checker's planes after put / add of `blocks` (block i of the stream where live[i])"""
        out = []
        for p, (idx, off) in enumerate(self.block_offsets()):
            if live is not None:
                keep = live[idx]
                idx, off = idx[keep], off[keep]
            out.append(orc_idct8(kind, blocks[idx], self.buf[p], off, self.ls[p])[1])
        return out

    def device(self):
        import torch
        d = [torch.from_numpy(b).cuda() for b in self.buf]
        return d, [d[p].data_ptr() + self.org[p] for p in range(3)]

    def check(self, got, exp, what):
        for p in range(3):
            assert (exp[p][~self.mask[p]] == SENT).all()
            assert np.array_equal(got[p], exp[p]), f"{what}: plane {p}: {diff_report(got[p], exp[p], self.mask[p])}"


def tiled_expect(mb_w, mb_h, nf):
    best, _ = mb420_segs(mb_w)
    grid_x = -(-((mb_w + 7) // 8) // best)
    return [((grid_x, mb_h, min(65535, nf - f0)), (48 * best, 1, 1)) for f0 in range(0, nf, 65535)]


def _mb420_cases():
    cs = []
    for kind in (1, 2):
        k = KIND_NAMES[kind]
        for w in MB420_WIDTHS:
            cs.append(pytest.param("tiled", kind, w, mb420_height(w), 2, {}, id=f"tiled-{width_id(w)}-{k}"))
        cs.append(pytest.param("tiled", kind, 240, 135, 1, {}, id=f"tiled-4k-240x135-{k}"))
        cs.append(pytest.param("tiled", kind, 1, 1, 65539, dict(pad=(16, 8, 8)), id=f"tiled-frames65539-{k}"))
        for tag, kw in (("luma-ls8mod16", dict(pad=(8, 16, 16))), ("chroma-ls-odd", dict(pad=(32, 9, 16))),
                        ("luma-plane+1", dict(shift=(1, 0, 0))), ("chroma-plane+1", dict(shift=(0, 0, 1))),
                        ("bottomup", dict(bottom_up=True))):
            cs.append(pytest.param("warp", kind, 17, 4, 2, kw, id=f"warp-{tag}-{k}"))
        cs.append(pytest.param("warp", kind, 1, 65536, 1, dict(pad=(16, 8, 8)), id=f"warp-mbh65536-{k}"))
    return cs


@pytest.mark.parametrize("route, kind, mb_w, mb_h, nf, layout", _mb420_cases())
def test_mb420_route(device, route, kind, mb_w, mb_h, nf, layout):
    import torch
    from ffmpeg_b200 import idctdsp
    n = mb_w * mb_h * 6 * nf
    blocks, _ = mixed_blocks(n, mb_w * 1000 + mb_h + nf + kind)
    pics = Pics(mb_w, mb_h, nf, mb_w + kind, **layout)
    exp = pics.oracle(kind, blocks)
    with on_stream(device):
        db = torch.from_numpy(blocks).cuda()
        dp, _ = pics.device()
        call = lambda b, *p: idctdsp.idct_mb420_device(device, kind, b, mb_w, mb_h, nf, [t.data_ptr() + o for t, o in zip(p, pics.org)],  # noqa: E731
                                                      pics.ls, pics.fs)
        call(db, *dp)
        device.sync()
        got = [t.cpu().numpy() for t in dp]
        assert np.array_equal(db.cpu().numpy(), blocks), "the coefficient stream changed"
    pics.check(got, exp, f"{route} {KIND_NAMES[kind]}")


# ---------------------------------------------------------------------------------------------- thread-per-block batches
def uniform_layout(n, line_size, elem, rng, bottom_up=False):
    """block i at a random column of one picture of 8 rows, |line_size| bytes apart: (byte offsets, buffer size)"""
    a = abs(line_size)
    off = HEAD + rng.permutation(n).astype(np.int64) * 8 * elem + 7 * a * bottom_up
    return off, HEAD + 8 * a + TAIL


def dest_buffer(size, off, ls, elem, rng, maxv=255):
    """SENT everywhere but the blocks' rows, which hold random samples below maxv + 1; and the mask of those rows' bytes"""
    buf = np.full(size, SENT, np.uint8)
    pos = footprint(off, ls, 8, elem)
    if elem == 1:
        buf[pos] = rng.integers(0, maxv + 1, pos.size, dtype=np.uint8)
    else:
        s = footprint(off // 2, np.asarray(ls) // 2, 8, 1)
        buf.view(np.uint16)[s] = rng.integers(0, maxv + 1, s.size, dtype=np.uint16)
    mask = np.zeros(size, bool)
    mask[pos] = True
    return buf, mask


def run_tpb(device, kind, blocks, buf, off, ls_arr, uniform, blk_shift=0, extra_blocks=4):
    """b200_idct_batch_device on blocks (followed by `extra_blocks` sentinel blocks): (blocks buffer after, dest after)"""
    import torch
    from ffmpeg_b200 import idctdsp
    n = blocks.shape[0]
    cbuf = np.full((n + extra_blocks) * 128 + blk_shift + TAIL, SENT, np.uint8)
    cbuf[blk_shift:blk_shift + n * 128] = blocks.view(np.uint8).ravel()
    with on_stream(device):
        dc = torch.from_numpy(cbuf).cuda()
        dd = torch.from_numpy(buf).cuda() if buf is not None else None
        do = torch.from_numpy(off).cuda() if off is not None else None
        dl = torch.from_numpy(np.ascontiguousarray(ls_arr, np.int32)).cuda() if ls_arr is not None else None
        call = lambda c, d, o, ls: idctdsp.idct_batch_device(device, kind, c.data_ptr() + blk_shift, n, d, o, ls, uniform)  # noqa: E731
        call(dc, dd, do, dl)
        device.sync()
        return dc.cpu().numpy(), dd.cpu().numpy() if dd is not None else None


def check_tpb(n, kind, cbuf, blocks, expb, got, exp, mask):
    after = cbuf[:n * 128].view(np.int16).reshape(n, 64)
    assert (cbuf[n * 128:] == SENT).all(), "bytes past the last block changed"
    if kind == 0:
        bad = np.nonzero((after != expb).any(axis=1))[0]
        assert not len(bad), f"{len(bad)} blocks differ from the checker, first {bad[:8].tolist()}"
    else:
        assert np.array_equal(after, blocks), "the coefficients changed"
        assert np.array_equal(got, exp), diff_report(got, exp, mask)


TPB_COUNTS = (1, 127, 128, 129, 255, 257, 100_003)


@pytest.mark.parametrize("n, kind", [pytest.param(n, k, id=f"tpb-{KIND_NAMES[k]}-n{n}") for k in (0, 1, 2) for n in TPB_COUNTS])
def test_tpb_counts(device, n, kind):
    """uniform line size, scattered destinations; kind 0 in place with sentinel blocks after nblocks"""
    rng = np.random.default_rng([n, kind])
    blocks, _ = mixed_blocks(n, n + kind)
    if kind == 0:
        expb, _ = orc_idct8(0, blocks, None, None, 0)
        cbuf, _ = run_tpb(device, 0, blocks, None, None, None, 0)
        check_tpb(n, 0, cbuf, blocks, expb, None, None, None)
        return
    ls = 8 * n + 8
    off, size = uniform_layout(n, ls, 1, rng)
    buf, mask = dest_buffer(size, off, ls, 1, rng)
    _, exp = orc_idct8(kind, blocks, buf, off, ls)
    cbuf, got = run_tpb(device, kind, blocks, buf, off, None, ls)
    check_tpb(n, kind, cbuf, blocks, None, got, exp, mask)


@pytest.mark.parametrize("layout, kind", [pytest.param(lay, k, id=f"tpb-{lay}-{KIND_NAMES[k]}") for k in (1, 2)
                                          for lay in ("lsarray-aligned", "lsarray-unaligned", "oddls-aligned")])
def test_tpb_line_sizes(device, layout, kind):
    """per-block line sizes mixing positive, negative and odd values (dest 8-byte aligned or not), and a uniform odd line size
    with 8-byte aligned destinations: the byte path"""
    n = 257
    rng = np.random.default_rng([len(layout), kind])
    blocks, _ = mixed_blocks(n, 77 + kind)
    if layout.startswith("lsarray"):
        ls = np.array(LS8)[rng.integers(0, len(LS8), n)]
        shifts = np.zeros(n, np.int64) if layout.endswith("-aligned") else rng.choice([1, 3, 4, 5, 7], n)
        off, size = private_rows(ls, shifts)
        arr, uniform = ls, 0
    else:
        ls = 8 * n + 9
        off, size = uniform_layout(n, ls, 1, rng)
        arr, uniform = None, ls
    buf, mask = dest_buffer(size, off, ls, 1, rng)
    _, exp = orc_idct8(kind, blocks, buf, off, ls)
    cbuf, got = run_tpb(device, kind, blocks, buf, off, arr, uniform)
    check_tpb(n, kind, cbuf, blocks, None, got, exp, mask)


@pytest.mark.parametrize("kind", [0, 1, 2], ids=lambda k: f"tpb-refuse-blocks+8-{KIND_NAMES[k]}")
def test_tpb_refuses_blocks_not_16_byte_aligned(device, kind):
    import ffmpeg_b200 as fb
    n = 40
    rng = np.random.default_rng(kind)
    blocks, _ = mixed_blocks(n, 5)
    off, size = uniform_layout(n, 8 * n, 1, rng)
    buf, _ = dest_buffer(size, off, 8 * n, 1, rng)
    before = launch_count()
    with pytest.raises(fb.B200Error):
        run_tpb(device, kind, blocks, buf if kind else None, off if kind else None, None, 8 * n, blk_shift=8)
    assert launch_count() == before


# ---------------------------------------------------------------------------------------------- fused quantiser + IDCT
def fused_inputs(variant, n, seed):
    """cl.unquant_case's decoder-like blocks and parameters, half of the blocks replaced by the ten classes as levels"""
    cfg, ub, _, q, last = cl.unquant_case(seed, variant, nblocks=n)
    cb, _ = mixed_blocks(n, seed)
    pick = np.random.default_rng(seed).random(n) < 0.5
    return cfg, np.where(pick[:, None], cb, ub).astype(np.int16), q, last


def run_fused(device, variant, cfg, kind, blocks, q, last, pics):
    import torch
    from ffmpeg_b200 import mpegvideo
    from ffmpeg_b200._lib import MpvUnquant
    params = cl.unquant_params(struct=MpvUnquant, **cfg)
    with on_stream(device):
        db = torch.from_numpy(blocks).cuda()
        dq, dl = torch.from_numpy(q).cuda(), torch.from_numpy(last).cuda()
        dp, _ = pics.device()
        call = lambda b, *p: mpegvideo.unquant_idct_mb420_device(device, variant, params, kind, b, dq, dl, pics.mb_w, pics.mb_h,  # noqa: E731
                                                                 pics.nf, [t.data_ptr() + o for t, o in zip(p, pics.org)], pics.ls, pics.fs)
        call(db, *dp)
        device.sync()
        assert np.array_equal(db.cpu().numpy(), blocks), "the coefficient stream changed"
        return [t.cpu().numpy() for t in dp]


def fused_oracle(variant, cfg, kind, blocks, q, last, pics):
    deq = cl.orc_unquant(variant, cfg, blocks, None, q, last)                      # block number inside the macroblock = i % 6
    return pics.oracle(kind, deq, (last >= 0) if kind == 2 else None)               # add_dequant_dct skips last_index < 0


@pytest.mark.parametrize("mb_w, kind", [pytest.param(w, k, id=f"fused-{width_id(w)}-{KIND_NAMES[k]}") for k in (1, 2) for w in MB420_WIDTHS])
def test_fused_widths(device, mb_w, kind):
    mb_h, nf = mb420_height(mb_w), 2
    n = mb_w * mb_h * 6 * nf
    for variant in range(7):
        cfg, blocks, q, last = fused_inputs(variant, n, 4000 + mb_w * 7 + variant)
        pics = Pics(mb_w, mb_h, nf, variant + kind)
        got = run_fused(device, variant, cfg, kind, blocks, q, last, pics)
        pics.check(got, fused_oracle(variant, cfg, kind, blocks, q, last, pics), cl.UNQUANT_VARIANTS[variant])


@pytest.mark.parametrize("kind", [1, 2], ids=lambda k: KIND_NAMES[k])
@pytest.mark.parametrize("variant", range(7), ids=lambda v: f"fused-extreme-{cl.UNQUANT_VARIANTS[v]}")
def test_fused_extreme(device, variant, kind):
    """full-range levels, qscale 1 and 31 with both q_scale_type, matrices up to 255, DC products that wrap int16, h263_aic and
    ac_pred both ways, last_index 0 / 63 (and -1 for the MPEG variants)"""
    mb_w, mb_h, nf = 41, 2, 2
    n = mb_w * mb_h * 6 * nf
    for i, (qt, aic, acp) in enumerate(extreme_configs()):
        cfg, blocks, _, q, last = extreme_unquant_case(30 + i, variant, n, qt, aic, acp)
        pics = Pics(mb_w, mb_h, nf, i)
        got = run_fused(device, variant, cfg, kind, blocks, q, last, pics)
        pics.check(got, fused_oracle(variant, cfg, kind, blocks, q, last, pics), (cl.UNQUANT_VARIANTS[variant], qt, aic, acp))


@pytest.mark.parametrize("kind", [1, 2], ids=lambda k: f"fused-1080p-vs-two-kernels-{KIND_NAMES[k]}")
def test_fused_equals_two_kernels_1080p(device, kind):
    """put_dct / add_dequant_dct in one kernel = unquantize_batch_device followed by idct_mb420_device on the same inputs (add: only
    blocks with last_index >= 0 reach the quantiser, as in the decoder)"""
    import torch
    from ffmpeg_b200 import idctdsp, mpegvideo
    from ffmpeg_b200._lib import MpvUnquant
    mb_w, mb_h, nf = 120, 68, 1
    n = mb_w * mb_h * 6 * nf
    for variant in range(7):
        cfg, blocks, q, last = fused_inputs(variant, n, 900 + variant)
        if kind == 2:
            last = np.maximum(last, 0).astype(np.int8)
        pics = Pics(mb_w, mb_h, nf, 50 + variant)
        fused = run_fused(device, variant, cfg, kind, blocks, q, last, pics)
        with on_stream(device):
            db = torch.from_numpy(blocks).cuda()
            dq, dl = torch.from_numpy(q).cuda(), torch.from_numpy(last).cuda()
            dp, planes = pics.device()
            mpegvideo.unquantize_batch_device(device, variant, cl.unquant_params(struct=MpvUnquant, **cfg), db, n, None, dq, dl)
            idctdsp.idct_mb420_device(device, kind, db, mb_w, mb_h, nf, planes, pics.ls, pics.fs)
            device.sync()
            two = [t.cpu().numpy() for t in dp]
        for p in range(3):
            assert np.array_equal(fused[p], two[p]), (cl.UNQUANT_VARIANTS[variant], p, int((fused[p] != two[p]).sum()))
        pics.check(fused, fused_oracle(variant, cfg, kind, blocks, q, last, pics), cl.UNQUANT_VARIANTS[variant])


@pytest.mark.parametrize("what", ["frames65536", "unaligned", "bottomup", "not-a-permutation"], ids=lambda w: f"fused-refuse-{w}")
def test_fused_refusals_change_nothing(device, what):
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import mpegvideo
    from ffmpeg_b200._lib import MpvUnquant
    mb_w, mb_h, nf = (1, 1, 65536) if what == "frames65536" else (17, 2, 1)
    n = mb_w * mb_h * 6 * nf
    layout = {"unaligned": dict(shift=(0, 1, 0)), "bottomup": dict(bottom_up=True)}.get(what, {})
    pics = Pics(mb_w, mb_h, nf, 3, **layout)
    blocks, _ = mixed_blocks(n, 8)
    q = np.full(n, 5, np.uint8)
    last = np.full(n, 63, np.int8)
    with on_stream(device):
        db = torch.from_numpy(blocks).cuda()
        dq, dl = torch.from_numpy(q).cuda(), torch.from_numpy(last).cuda()
        dp, planes = pics.device()
        for variant in range(7):
            cfg = cl.unquant_case(variant, variant, nblocks=8)[0]
            params = cl.unquant_params(struct=MpvUnquant, **cfg)
            if what == "not-a-permutation":
                params.permutated[9] = params.permutated[10]
            for kind in (1, 2):
                before = launch_count()
                with pytest.raises(fb.B200Error):
                    mpegvideo.unquant_idct_mb420_device(device, variant, params, kind, db, dq, dl, mb_w, mb_h, nf, planes, pics.ls, pics.fs)
                assert launch_count() == before, (cl.UNQUANT_VARIANTS[variant], kind)
        device.sync()
        for p in range(3):
            assert np.array_equal(dp[p].cpu().numpy(), pics.buf[p]), p
        assert np.array_equal(db.cpu().numpy(), blocks)


# ---------------------------------------------------------------------------------------------- standalone inverse quantiser
def run_unquant(device, variant, cfg, blocks, blk_n, q, last, shift=0):
    """blocks placed `shift` bytes past a 16-byte boundary, SENT before and after: (blocks after, whole buffer)"""
    import torch
    from ffmpeg_b200 import mpegvideo as mv
    from ffmpeg_b200._lib import MpvUnquant
    n = blocks.shape[0]
    buf = np.full(HEAD + shift + n * 128 + TAIL, SENT, np.uint8)
    buf[HEAD + shift:HEAD + shift + n * 128] = blocks.view(np.uint8).ravel()
    p = cl.unquant_params(struct=MpvUnquant, **cfg)
    with on_stream(device):
        d = torch.from_numpy(buf).cuda()
        dn = torch.from_numpy(blk_n).cuda() if blk_n is not None else None
        dq, dl = torch.from_numpy(q).cuda(), torch.from_numpy(last).cuda()
        call = lambda b: mv.unquantize_batch_device(device, variant, p, b.data_ptr() + HEAD + shift, n, dn, dq, dl)  # noqa: E731
        call(d)
        device.sync()
        out = d.cpu().numpy()
    return out[HEAD + shift:HEAD + shift + n * 128].copy().view(np.int16).reshape(n, 64), out


def check_unquant_buffer(out, shift, n):
    assert (out[:HEAD + shift] == SENT).all() and (out[HEAD + shift + n * 128:] == SENT).all(), "bytes around the blocks changed"


UNQUANT_LOOP_N = 150_001


@pytest.mark.parametrize("blkn", [True, False], ids=["blkn", "mbstream"])
@pytest.mark.parametrize("variant", range(7), ids=lambda v: f"unquant-loop-{cl.UNQUANT_VARIANTS[v]}")
def test_unquant_warps_loop(device, variant, blkn):
    """150,001 blocks: more than four per warp of the capped grid, so every warp walks several blocks"""
    n = UNQUANT_LOOP_N
    rng = np.random.default_rng([variant, blkn])
    cfg = cl.unquant_case(70 + variant, variant, nblocks=8)[0]
    blocks, _ = mixed_blocks(n, 70 + variant)
    q = rng.integers(1, 32, n).astype(np.uint8)
    last = rng.integers(0 if variant in H263 else -1, 64, n).astype(np.int8)
    blk_n = rng.integers(0, 6, n).astype(np.uint8) if blkn else None
    got, out = run_unquant(device, variant, cfg, blocks, blk_n, q, last)
    exp = cl.orc_unquant(variant, cfg, blocks, blk_n, q, last)
    bad = np.nonzero((got != exp).any(axis=1))[0]
    assert not len(bad), f"{len(bad)} blocks differ from the checker, first {bad[:8].tolist()}"
    check_unquant_buffer(out, 0, n)


@pytest.mark.parametrize("variant", range(7), ids=lambda v: f"unquant-offset4-{cl.UNQUANT_VARIANTS[v]}")
def test_unquant_blocks_4_byte_aligned(device, variant):
    n = 1001
    rng = np.random.default_rng(variant)
    cfg = cl.unquant_case(90 + variant, variant, nblocks=8)[0]
    blocks, _ = mixed_blocks(n, 90 + variant)
    q = rng.integers(1, 32, n).astype(np.uint8)
    last = rng.integers(0 if variant in H263 else -1, 64, n).astype(np.int8)
    for shift, blk_n in ((4, rng.integers(0, 6, n).astype(np.uint8)), (12, None)):
        got, out = run_unquant(device, variant, cfg, blocks, blk_n, q, last, shift=shift)
        assert np.array_equal(got, cl.orc_unquant(variant, cfg, blocks, blk_n, q, last)), (shift, blk_n is None)
        check_unquant_buffer(out, shift, n)


@pytest.mark.parametrize("variant", range(7), ids=lambda v: f"unquant-extreme-{cl.UNQUANT_VARIANTS[v]}")
def test_unquant_extreme(device, variant):
    for i, (qt, aic, acp) in enumerate(extreme_configs()):
        cfg, blocks, blk_n, q, last = extreme_unquant_case(50 + i, variant, 600, qt, aic, acp)
        use_n = blk_n if i & 1 else None
        got, out = run_unquant(device, variant, cfg, blocks, use_n, q, last)
        assert np.array_equal(got, cl.orc_unquant(variant, cfg, blocks, use_n, q, last)), (qt, aic, acp)
        check_unquant_buffer(out, 0, blocks.shape[0])


# ---------------------------------------------------------------------------------------------- 10 / 12 bit and ProRes
HBD_COUNTS = (1, 127, 128, 129, 255, 257)


def hbd_layout(layout, n, rng):
    """(byte offsets, line sizes: int or per-block array, buffer size, per-block array to pass or None, uniform line size)"""
    if layout != "lsarray":
        ls = {"rows16": 16 * n + 32, "uniform": 16 * n + 32, "samples": 16 * n + 18, "bottomup": -(16 * n + 32)}[layout]
        off, size = uniform_layout(n, ls, 2, rng, bottom_up=ls < 0)
        return off, ls, size, None, ls
    ls = np.array(LS16)[rng.integers(0, len(LS16), n)]
    off, size = private_rows(ls, 2 * rng.integers(0, 8, n), elem=2)
    return off, ls, size, ls, 0


def run_hbd_like(device, fn, blocks, buf, off, arr, qmat=None):
    """fn(coefficients, dest, dest_off, line_size array, qmat) on device copies: (coefficient buffer after, dest after)"""
    import torch
    n = blocks.shape[0]
    cbuf = np.full((n + 4) * 128 + TAIL, SENT, np.uint8)
    cbuf[:n * 128] = blocks.view(np.uint8).ravel()
    with on_stream(device):
        dc = torch.from_numpy(cbuf).cuda()
        dd = torch.from_numpy(buf).cuda() if buf is not None else None
        do = torch.from_numpy(off).cuda() if off is not None else None
        dl = torch.from_numpy(np.ascontiguousarray(arr, np.int32)).cuda() if arr is not None else None
        dqm = torch.from_numpy(qmat).cuda() if qmat is not None else None
        fn(dc, dd, do, dl, dqm)
        device.sync()
        return dc.cpu().numpy(), dd.cpu().numpy() if dd is not None else None


def _hbd_cases():
    cs = []
    for depth in (9, 10, 12):
        cs.append(pytest.param(depth, 0, "inplace", id=f"hbd-d{depth}-idct-inplace"))
        for kind in (1, 2):
            for layout in ("rows16", "samples", "lsarray", "bottomup"):
                cs.append(pytest.param(depth, kind, layout, id=f"hbd-d{depth}-{KIND_NAMES[kind]}-{layout}"))
    return cs


@pytest.mark.parametrize("depth, kind, layout", _hbd_cases())
def test_hbd_route(device, depth, kind, layout):
    from ffmpeg_b200 import idctdsp
    maxv = (1 << (12 if depth == 12 else 10)) - 1
    for n in HBD_COUNTS if layout != "lsarray" else (128, 257):
        rng = np.random.default_rng([depth, kind, n, len(layout)])
        blocks, _ = mixed_blocks(n, depth * 100 + n)
        if kind == 0:
            expb, _ = orc_hbd(depth, 0, blocks, np.zeros(16, np.uint8), np.zeros(n, np.int64), 0)
            cbuf, _ = run_hbd_like(device, lambda dc, dd, do, dl, qm: idctdsp.idct_hbd_batch_device(device, depth, 0, dc, n),
                                       blocks, None, None, None)
            assert np.array_equal(cbuf[:n * 128].view(np.int16).reshape(n, 64), expb), n
        else:
            off, ls, size, arr, uniform = hbd_layout(layout, n, rng)
            buf, mask = dest_buffer(size, off, ls, 2, rng, maxv)
            _, exp = orc_hbd(depth, kind, blocks, buf, off, ls)
            cbuf, got = run_hbd_like(device, lambda dc, dd, do, dl, qm: idctdsp.idct_hbd_batch_device(device, depth, kind, dc, n, dd, do, dl,
                                                                                                           uniform),
                                         blocks, buf, off, arr)
            assert np.array_equal(cbuf[:n * 128].view(np.int16).reshape(n, 64), blocks), (n, "the coefficients changed")
            assert np.array_equal(got, exp), (n, diff_report(got, exp, mask))
        assert (cbuf[n * 128:] == SENT).all(), (n, "bytes past the last block changed")


@pytest.mark.parametrize("bits, layout", [pytest.param(b, lay, id=f"prores-b{b}-{lay}") for b in (10, 12)
                                          for lay in ("uniform", "lsarray", "bottomup")])
def test_prores_route(device, bits, layout):
    """quantiser matrices up to 255 on full-range levels: the products wrap int16"""
    from ffmpeg_b200 import idctdsp
    for n in (1, 127, 128, 129, 257):
        rng = np.random.default_rng([bits, n, len(layout)])
        blocks, _ = mixed_blocks(n, bits * 100 + n)
        qmat = prores_qmat(n + bits)
        off, ls, size, arr, uniform = hbd_layout(layout, n, rng)
        buf, mask = dest_buffer(size, off, ls, 2, rng, (1 << bits) - 1)
        _, exp = orc_prores(bits, blocks, qmat, buf, off, ls)
        cbuf, got = run_hbd_like(device, lambda dc, dd, do, dl, qm: idctdsp.prores_idct_put_batch_device(device, bits, dc, n, qm, dd, do, dl,
                                                                                                             uniform),
                                     blocks, buf, off, arr, qmat)
        assert np.array_equal(cbuf[:n * 128].view(np.int16).reshape(n, 64), blocks), (n, "the coefficients changed")
        assert (cbuf[n * 128:] == SENT).all(), (n, "bytes past the last block changed")
        assert np.array_equal(got, exp), (n, diff_report(got, exp, mask))


# ---------------------------------------------------------------------------------------------- which kernel each route launches
# The cases above check results; these check that each case shape reaches the kernel, grid and block its route names.  The launches
# are read from torch.profiler, in one session in a child process: the profiler's state (it can miss the first kernels of a
# session, more often after many sessions) then stays out of the process that runs the rest of the suite.
ROUTES = ("tiled", "warp", "tpb", "fused", "unquant", "hbd", "prores")


def _route_table(sm_count):
    """[(case id, kernel, [(grid, block)] per launch, make)]: make(device) allocates buffers of the case's shape (contents do not
    choose the route) and returns the call"""
    rows = []
    tpb = lambda n: [((-(-n // 128), 1, 1), (128, 1, 1))]                                                      # noqa: E731
    for p in _mb420_cases():
        route, kind, mb_w, mb_h, nf, layout = p.values
        n = mb_w * mb_h * 6 * nf
        if route == "tiled":
            rows.append((p.id, "idct_mb420_kernel", tiled_expect(mb_w, mb_h, nf), ("mb420", kind, mb_w, mb_h, nf, layout)))
        else:
            rows.append((p.id, "idct8x8_kernel", [((-(-n // 32), 1, 1), (256, 1, 1))], ("mb420", kind, mb_w, mb_h, nf, layout)))
    for kind in (1, 2):
        for w in MB420_WIDTHS:
            rows.append((f"fused-{width_id(w)}-{KIND_NAMES[kind]}", "idct_mb420_kernel", tiled_expect(w, mb420_height(w), 2),
                         ("fused", kind, w, mb420_height(w), 2)))
    for kind in (0, 1, 2):
        for n in TPB_COUNTS:
            rows.append((f"tpb-{KIND_NAMES[kind]}-n{n}", "idct_tpb_kernel", tpb(n), ("tpb", kind, n, None)))
    for kind in (1, 2):
        for lay in ("lsarray-aligned", "lsarray-unaligned", "oddls-aligned"):
            rows.append((f"tpb-{lay}-{KIND_NAMES[kind]}", "idct_tpb_kernel", tpb(257), ("tpb", kind, 257, lay)))
    cap = sm_count * 16 * 8
    assert 4 * cap < UNQUANT_LOOP_N                                              # every warp walks more than one block
    for v in range(7):
        rows.append((f"unquant-loop-{cl.UNQUANT_VARIANTS[v]}", "mpv_unquant_kernel", [((min(cap, -(-UNQUANT_LOOP_N // 4)), 1, 1), (128, 1, 1))],
                     ("unquant", v, UNQUANT_LOOP_N)))
    for depth in (9, 10, 12):
        for kind, layout in [(0, "inplace")] + [(k, lay) for k in (1, 2) for lay in ("rows16", "samples", "lsarray", "bottomup")]:
            for n in (1, 257):
                rows.append((f"hbd-d{depth}-{KIND_NAMES[kind]}-{layout}-n{n}", "idct_hbd_kernel", tpb(n), ("hbd", depth, kind, layout, n)))
    for bits in (10, 12):
        for layout in ("uniform", "lsarray", "bottomup"):
            for n in (1, 257):
                rows.append((f"prores-b{bits}-{layout}-n{n}", "prores_idct_put_kernel", tpb(n), ("prores", bits, layout, n)))
    return rows


def _make_call(device, spec):
    """device buffers for one row of _route_table and the call that uses them"""
    import torch
    from ffmpeg_b200 import idctdsp, mpegvideo
    from ffmpeg_b200._lib import MpvUnquant
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None                  # noqa: E731
    what, rng = spec[0], np.random.default_rng(0)
    if what in ("mb420", "fused"):
        kind, mb_w, mb_h, nf = spec[1:5]
        pics = Pics(mb_w, mb_h, nf, 0, **(spec[5] if what == "mb420" else {}))
        n = mb_w * mb_h * 6 * nf
        db, dp = cuda(np.zeros((n, 64), np.int16)), [cuda(b) for b in pics.buf]
        planes = [t.data_ptr() + o for t, o in zip(dp, pics.org)]
        if what == "mb420":
            return lambda: idctdsp.idct_mb420_device(device, kind, db, mb_w, mb_h, nf, planes, pics.ls, pics.fs)
        params = cl.unquant_params(struct=MpvUnquant, **cl.unquant_case(0, 0, nblocks=8)[0])
        dq, dl = cuda(np.ones(n, np.uint8)), cuda(np.full(n, 63, np.int8))
        return lambda: mpegvideo.unquant_idct_mb420_device(device, 0, params, kind, db, dq, dl, mb_w, mb_h, nf, planes, pics.ls, pics.fs)
    if what == "tpb":
        kind, n, lay = spec[1:]
        db = cuda(np.zeros((n, 64), np.int16))
        if kind == 0:
            return lambda: idctdsp.idct_batch_device(device, 0, db, n)
        if lay is None or lay.startswith("oddls"):
            ls = 8 * n + (9 if lay else 8)
            off, size = uniform_layout(n, ls, 1, rng)
            arr, uniform = None, ls
        else:
            arr = np.array(LS8)[rng.integers(0, len(LS8), n)]
            off, size = private_rows(arr, np.zeros(n, np.int64) if lay.endswith("-aligned") else rng.choice([1, 3, 4, 5, 7], n))
            uniform = 0
        dd, do, dl = cuda(np.zeros(size, np.uint8)), cuda(off), cuda(None if arr is None else arr.astype(np.int32))
        return lambda: idctdsp.idct_batch_device(device, kind, db, n, dd, do, dl, uniform)
    if what == "unquant":
        v, n = spec[1:]
        params = cl.unquant_params(struct=MpvUnquant, **cl.unquant_case(0, v, nblocks=8)[0])
        db, dq, dl = cuda(np.zeros((n, 64), np.int16)), cuda(np.ones(n, np.uint8)), cuda(np.full(n, 63, np.int8))
        return lambda: mpegvideo.unquantize_batch_device(device, v, params, db, n, None, dq, dl)
    if what == "hbd":
        depth, kind, layout, n = spec[1:]
        db = cuda(np.zeros((n, 64), np.int16))
        if kind == 0:
            return lambda: idctdsp.idct_hbd_batch_device(device, depth, 0, db, n)
        off, ls, size, arr, uniform = hbd_layout(layout, n, rng)
        dd, do, dl = cuda(np.zeros(size, np.uint8)), cuda(off), cuda(None if arr is None else arr.astype(np.int32))
        return lambda: idctdsp.idct_hbd_batch_device(device, depth, kind, db, n, dd, do, dl, uniform)
    bits, layout, n = spec[1:]
    off, ls, size, arr, uniform = hbd_layout(layout, n, rng)
    db, dq = cuda(np.zeros((n, 64), np.int16)), cuda(prores_qmat(1))
    dd, do, dl = cuda(np.zeros(size, np.uint8)), cuda(off), cuda(None if arr is None else arr.astype(np.int32))
    return lambda: idctdsp.prores_idct_put_batch_device(device, bits, db, n, dq, dd, do, dl, uniform)


def record_routes(path, tries=3):
    """Child process: every call of _route_table in one torch.profiler session, a spin kernel after each (and three before the
    first) on the library's stream; writes {case id: [(kernel, grid, block)]} of the library's kernels to `path`."""
    import torch
    import ffmpeg_b200 as fb
    from torch.profiler import ProfilerActivity, profile
    dev = fb.Device(0)
    dev.set_default()
    rows = _route_table(torch.cuda.get_device_properties(0).multi_processor_count)
    groups = []
    with on_stream(dev):
        for _ in range(tries):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    torch.cuda._sleep(100_000)
                for row in rows:
                    call = _make_call(dev, row[3])
                    call()
                    torch.cuda._sleep(1000)
                    del call
                dev.sync()
                torch.cuda.synchronize()
            with tempfile.TemporaryDirectory() as d:
                trace = os.path.join(d, "trace.json")
                prof.export_chrome_trace(trace)
                with open(trace) as f:
                    events = json.load(f)["traceEvents"]
            ks = [(e["name"], e["args"]["grid"], e["args"]["block"]) for e in sorted(events, key=lambda e: e.get("ts", 0))
                  if e.get("cat") == "kernel" and ("spin_kernel" in e["name"] or "at::" not in e["name"])]
            while ks and "spin_kernel" in ks[0][0]:                               # the leading spins, however many were recorded
                ks.pop(0)
            groups, cur = [], []
            for k in ks:
                if "spin_kernel" in k[0]:
                    groups.append(cur)
                    cur = []
                else:
                    cur.append(k)
            if len(groups) == len(rows) and not cur:
                break
    dev.close()
    with open(path, "w") as f:
        json.dump({row[0]: g for row, g in zip(rows, groups)} if len(groups) == len(rows) else {}, f)


@pytest.fixture(scope="module")
def recorded_routes(device):
    import subprocess
    import sys
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    here = os.path.dirname(os.path.abspath(__file__))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "routes.json")
        code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; import test_idct_routes_gpu as T; "
                f"T.record_routes({path!r})")
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, "route recording failed:\n" + r.stdout[-3000:] + r.stderr[-3000:]
        with open(path) as f:
            got = json.load(f)
    assert got, "torch.profiler did not record the route calls whole"
    return got, torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("route", ROUTES, ids=lambda r: f"{r}-launches")
def test_route_launches(recorded_routes, route):
    """every case shape of the route launches only the route's kernel, with the grid and block the dispatcher must pick"""
    got, sm_count = recorded_routes
    bad = []
    for cid, name, expect, _ in _route_table(sm_count):
        if cid.split("-")[0] != route:
            continue
        ks = got[cid]
        if any(name not in k[0] for k in ks) or [(tuple(k[1]), tuple(k[2])) for k in ks] != expect:
            bad.append(f"{cid}: launched {[(k[0][:40], k[1], k[2]) for k in ks]}, expected {name} {expect}")
    assert not bad, f"{len(bad)} cases: " + "; ".join(bad[:6])
