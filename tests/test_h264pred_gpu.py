"""GPU tier for H.264 intra prediction (ffmpeg_b200/csrc/h264pred.cu) on the H100: both batched entries against the checker and the
reference's fixture hashes at every depth and chroma format, ops with invalid kinds, offsets beyond 2^31 bytes, and every drop-in
member of H264PredContext through host pointers.  Test ids start with the table (or entry) they exercise."""
import numpy as np
import pytest

import h264predlib as hp
from test_h264pred import DEPTHS, CODEC_H264, fixture_hashes, digest, run_members, member_of, field_case, checker_field

pytestmark = pytest.mark.gpu

PRED_NAMES = ["pred4x4", "pred8x8l", "pred8x8", "pred8x16", "pred16x16"]
ADD_NAMES = ["pred4x4_add", "pred8x8l_add", "pred8x8l_filter_add", "pred8x8_add", "pred8x16_add", "pred16x16_add"]


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def on_device(dev, depth, add, pic, kinds, flags, off, coef, coef_off):
    """one batched call on device copies of a case; returns (picture, coefficients) as numpy"""
    import torch
    from ffmpeg_b200 import pel
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()
        dp, dk, df, do, dc, dco = t(pic), t(kinds), t(flags), t(off), t(coef), t(coef_off)
        if add:
            pel.h264_pred_add_batch_device(dev, depth, len(kinds), dk, df, dp, do, pic.strides[0], dc, dco)
        else:
            pel.h264_pred_batch_device(dev, depth, len(kinds), dk, df, dp, do, pic.strides[0])
        dev.sync()
        return dp.cpu().numpy().view(pic.dtype), dc.cpu().numpy()


def table_cases():
    for add, names in ((False, PRED_NAMES), (True, ADD_NAMES)):
        for t, name in enumerate(names):
            for depth in DEPTHS:
                yield pytest.param(add, t, depth, id=f"{name}-d{depth}")


@pytest.mark.parametrize("add,table,depth", list(table_cases()))
def test_table_vs_checker(dev, add, table, depth):
    """the ops of one table (every mode and flags value, every content class, three rounds): whole picture and coefficients equal the
    checker, so samples outside each block are untouched and the add forms clear exactly their coefficients"""
    idc = 2 if table == (4 if add else 3) else 1
    combos = [c for c in hp.h264pred_combos(idc, add) if c[0] == table]
    n = 3 * len(hp.PRED_CLASSES) * len(hp.h264pred_combos(idc, add))
    pic, kinds, flags, off, coef, coef_off = hp.h264pred_case(5000 + 31 * table + depth + 7 * add, n, depth, idc, add)
    sel = np.array([i for i in range(n) if (kinds[i] >> 4) == table])
    assert len(sel) >= len(combos) * len(hp.PRED_CLASSES)
    case = (pic, kinds[sel], flags[sel], off[sel], coef, coef_off[sel])
    got = on_device(dev, depth, add, *case)
    exp = hp.orc_h264pred(depth, idc, add, *case)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
    assert not np.array_equal(got[0], pic)


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("idc", (1, 2), ids=("420", "422"))
@pytest.mark.parametrize("add", (False, True), ids=("pred_batch", "pred_add_batch"))
def test_batch_vs_fixture(dev, add, idc, depth):
    """the seeded batch of every table behind tests/golden/h264pred_hashes.txt: the reference's picture and coefficients, bit for bit"""
    case = hp.h264pred_fixture_case(depth, idc, add)
    got = on_device(dev, depth, add, *case)
    assert digest(*got) == fixture_hashes()[(depth, idc, add)]


@pytest.mark.parametrize("add", (False, True), ids=("pred_batch", "pred_add_batch"))
def test_invalid_kinds_change_nothing(dev, add):
    bad = [(0, 2), (1, 3), (2, 2), (3, 0), (4, 0), (5, 0), (5, 3), (6, 1), (15, 15)] if add else \
          [(0, 12), (0, 15), (1, 12), (2, 11), (3, 15), (4, 7), (4, 8), (5, 0), (15, 15)]
    for depth in (8, 10):
        pic, kinds, flags, off, coef, coef_off = hp.h264pred_case(91, len(bad), depth, 1, add)
        kinds = np.array([(t << 4) | m for t, m in bad], np.uint8)
        got = on_device(dev, depth, add, pic, kinds, flags, off, coef, coef_off)
        assert np.array_equal(got[0], pic) and np.array_equal(got[1], coef)


@pytest.mark.parametrize("add", (False, True), ids=("pred16x16-beyond-2GiB", "pred16x16_add-beyond-2GiB"))
def test_offsets_beyond_2GiB(dev, add):
    """one call over a 2.2 GB picture: an op near the base and ops straddling and beyond the 2^31-byte mark; the rows around each
    op equal the checker, run on a copy of those rows"""
    import torch
    from ffmpeg_b200 import pel
    stride, rows = 4096, (1 << 31) // 4096 + 96
    rng = np.random.default_rng(5)
    y_ops = [8, (1 << 31) // stride - 8, (1 << 31) // stride + 40]
    kinds = np.array([(5 << 4) | 2, (5 << 4) | 1, (2 << 4) | 2] if add else [(4 << 4) | 3, (4 << 4) | 0, (1 << 4) | 4], np.uint8)
    flags = np.array([0, 0, 3], np.uint8)
    xs = [40, 2000, 4000]
    off = np.array([y * stride + x for y, x in zip(y_ops, xs)], np.int64)
    coef = rng.integers(-32768, 32768, (3, 256)).astype(np.int16)
    coef_off = np.arange(3, dtype=np.int64) * 256
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        d = torch.empty(rows * stride, dtype=torch.uint8, device="cuda")
        windows = []
        for y, x in zip(y_ops, xs):
            w = rng.integers(0, 256, (20, 64), dtype=np.uint8)          # rows y-2 .. y+17, columns x-16 .. x+47
            windows.append(w)
            for r in range(20):
                d[(y - 2 + r) * stride + x - 16:(y - 2 + r) * stride + x + 48] = torch.from_numpy(w[r]).cuda()
        dc = torch.from_numpy(coef).cuda()
        t = lambda a: torch.from_numpy(a).cuda()
        if add:
            pel.h264_pred_add_batch_device(dev, 8, 3, t(kinds), t(flags), d, t(off), stride, dc, t(coef_off))
        else:
            pel.h264_pred_batch_device(dev, 8, 3, t(kinds), t(flags), d, t(off), stride)
        dev.sync()
        got = [np.stack([d[(y - 2 + r) * stride + x - 16:(y - 2 + r) * stride + x + 48].cpu().numpy() for r in range(20)]) for y, x in zip(y_ops, xs)]
        gcoef = dc.cpu().numpy()
        del d
        torch.cuda.empty_cache()
    # the checker on each window: the op at (2, 16) of a 64-byte-stride copy
    wpic = np.concatenate(windows, 0)
    woff = np.array([(20 * i + 2) * 64 + 16 for i in range(3)], np.int64)
    exp, ecoef = hp.orc_h264pred(8, 1, add, wpic, kinds, flags, woff, coef, coef_off)
    assert np.array_equal(np.concatenate(got, 0), exp) and np.array_equal(gcoef, ecoef)
    assert not np.array_equal(exp, wpic)


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("idc", (1, 2), ids=("420", "422"))
def test_dropin_members(dev, depth, idc):
    """H264PredContext from ff_h264_pred_init through the library, every member it fills called with host pointers (pred4x4's topright
    in a separate buffer; the 8x8 / 8x16 / 16x16 add forms with frame and field block_offset tables) against the checker"""
    from ffmpeg_b200 import pel
    ctx = pel.ff_h264_pred_init(CODEC_H264, depth, idc)
    for add in (False, True):
        case = hp.h264pred_case(6000 + depth + 3 * idc + add, len(hp.PRED_CLASSES) * len(hp.h264pred_combos(idc, add)), depth, idc, add)
        got = run_members(ctx, depth, idc, add, *case)
        exp = hp.orc_h264pred(depth, idc, add, *case)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), add
    fc = field_case(depth, idc)
    got = run_members(ctx, depth, idc, True, *fc, field=True)
    exp = checker_field(depth, idc, *fc)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])


def smoke(dev):
    """smoke(): one small batched call per table of both entries at 8 and 10 bit, bit-compared with the checker"""
    for depth in (8, 10):
        for add in (False, True):
            for idc in (1, 2):
                combos = hp.h264pred_combos(idc, add)
                pic, kinds, flags, off, coef, coef_off = hp.h264pred_case(7 + depth + idc, len(combos), depth, idc, add)
                got = on_device(dev, depth, add, pic, kinds, flags, off, coef, coef_off)
                exp = hp.orc_h264pred(depth, idc, add, pic, kinds, flags, off, coef, coef_off)
                assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), ("h264 intra prediction mismatch", depth, add, idc)
