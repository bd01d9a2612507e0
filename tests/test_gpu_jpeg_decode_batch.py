"""jpeg.loadFromBytes for many files in one call (zb_jpeg_decode_batch): every file's status and pixels equal those of the single
call (zb_jpeg_decode), and so the oracle's wherever it decodes.  One batch mixes every colour layout, restart intervals, the serial
fallback, every pixel format and tiny to wide sizes; the same files in another order decode the same; 1024 copies of liza.jpg
(more than 65,535 reconstruction tiles); truncated, corrupted and refused files next to good ones, with the refused files'
destinations untouched; limits per file; two files whose bits pass 2^32 together; the argument errors; streams and threads; and
the Python mirror."""
import ctypes as C
import threading
from pathlib import Path

import numpy as np
import pytest

import jpeg_decode_oracle as jd
import jpeg_oracle as jo
import jpeg_streams as js
from test_gpu_jpeg_decode import BIG, _positions, _synthetic, content, zb_limits

pytestmark = pytest.mark.gpu

FIX = Path(__file__).resolve().parent / "golden" / "jpeg_decode"
SENTINEL = 0x5A


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def zb(torch):
    import zignal_b200 as zb
    return zb


def single(zb, data, pixfmt, limits=None):
    """(status, numpy pixels or None) of the single-file call."""
    try:
        return 0, zb.Image.decode_jpeg(data, pixfmt, limits).to_numpy()
    except zb.ZignalError as e:
        return e.status, None


def native(zb, data):
    try:
        return 0 if zb.jpeg_info(data).num_components == 1 else 2
    except zb.ZignalError:
        return 2


def shape_of(zb, data):
    try:
        h = zb.jpeg_info(data)
        return h.height, h.width
    except zb.ZignalError:
        return 4, 4


def raw_batch(zb, torch, datas, fmts, limits=None, dsts=None, stream=None):
    """zb_jpeg_decode_batch over sentinel-filled destinations: (return code, statuses, destination Images)."""
    n = len(datas)
    if dsts is None:
        dsts = []
        for d, f in zip(datas, fmts):
            img = zb.Image.init(*shape_of(zb, d), zb.PixFmt(f))
            img._t.fill_(SENTINEL)
            dsts.append(img)
    bufs = [(C.c_uint8 * max(1, len(d))).from_buffer_copy(d or b"\0") for d in datas]
    ptrs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    lens = (C.c_uint64 * n)(*[len(d) for d in datas])
    zimg = (zb.ZbImage * n)(*[x._zb() for x in dsts])
    fmt = (C.c_int * n)(*fmts)
    status = (C.c_int * n)()
    lim = None if limits is None else C.byref(limits._c())
    s = torch.cuda.current_stream().cuda_stream if stream is None else stream
    rc = zb.lib().zb_jpeg_decode_batch(n, ptrs, lens, lim, zimg, fmt, status, s)
    return rc, list(status), dsts


def assert_batch_equals_single(zb, torch, datas, fmts, limits=None, oracle=True):
    rc, status, dsts = raw_batch(zb, torch, datas, fmts, limits)
    assert rc == 0
    for k, (d, f) in enumerate(zip(datas, fmts)):
        want_rc, want = single(zb, d, f, limits)
        assert status[k] == want_rc, (k, status[k], want_rc)
        if want_rc == 0:
            assert np.array_equal(dsts[k].to_numpy(), want), k
            if oracle:
                assert np.array_equal(want, jd.decode(d, f, None if limits is None else _jd_limits(limits))), k
        elif want_rc != 31:   # refused on the host: the destination is untouched
            assert (dsts[k]._t == SENTINEL).all(), k
    return status


def _jd_limits(limits):
    return jd.Limits(**{f: getattr(limits, f) for f, _ in jd.Limits._fields_})


def mixed_set(zb):
    rng = np.random.default_rng(2024)
    datas = [(FIX / p.name).read_bytes() for p in sorted(FIX.glob("*.jpg"))]
    for sub in (0, 1, 2):
        datas.append(jo.encode(content(rng, 45, 67, 2), 85, sub))
    datas.append(jo.encode(content(rng, 45, 67, 0), 85))
    datas.append(zb.Image.from_numpy(content(rng, 40, 50, 2)).encode_jpeg(80, 1))   # 4:2:2
    for kind in ("411", "gray_id7_2x2", "gray_id1_2x2", "dri", "dri_ff_ends_scan", "flat_tables"):
        datas.append(_synthetic(kind, np.random.default_rng(len(kind))))
    for k, shape in enumerate([(1, 1), (1, 300), (300, 1), (17, 33), (16, 79), (16, 80), (16, 81), (2049, 17)]):
        datas.append(jo.encode(content(rng, shape[0], shape[1], 2), 90, k % 3))
    return datas


def test_mixed_batch_every_path(zb, torch):
    datas = mixed_set(zb)
    fmts = [k % 5 for k in range(len(datas))]
    status = assert_batch_equals_single(zb, torch, datas, fmts)
    assert status == [0] * len(datas)


def test_order_does_not_matter(zb, torch):
    datas = mixed_set(zb)
    fmts = [native(zb, d) for d in datas]
    perm = np.random.default_rng(7).permutation(len(datas))
    _, sa, da = raw_batch(zb, torch, datas, fmts)
    _, sb, db = raw_batch(zb, torch, [datas[i] for i in perm], [fmts[i] for i in perm])
    for j, i in enumerate(perm):
        assert sb[j] == sa[i] == 0
        assert np.array_equal(db[j].to_numpy(), da[i].to_numpy())


def test_1024_copies_of_liza(zb, torch):
    liza = (FIX / "liza.jpg").read_bytes()
    want = zb.Image.decode_jpeg(liza).to_numpy()
    assert np.array_equal(want, jd.decode(liza))
    out = zb.Image.decode_jpeg_batch([liza] * 1024)
    for img in out:
        assert isinstance(img, zb.Image)
        assert np.array_equal(img.to_numpy(), want)


def bad_files(zb):
    rng = np.random.default_rng(5)
    good = [jo.encode(content(rng, 61, 83, 2), 80, 2), (FIX / "pillow_restart4_420.jpg").read_bytes(),
            jo.encode(content(rng, 61, 83, 0), 80)]
    datas = list(good)
    for d in good:
        datas += [d[:cut] for cut in _positions(len(d), rng, d)[::3]]
    for d in good[:2]:
        start = d.index(b"\xFF\xDA") + 14
        for _ in range(12):
            b = bytearray(d)
            for i in rng.integers(start, len(b) - 2, 3):
                b[i] = int(rng.integers(0, 256))
            datas.append(bytes(b))
    datas += [c[0] for c in js.semantic_cases().values()]
    hdr = jo.encode(content(np.random.default_rng(1), 20, 20, 2), 90, 2)
    datas += [hdr[2:], hdr.replace(b"\xFF\xC0", b"\xFF\xC1", 1), hdr.replace(b"\xFF\xC0", b"\xFF\xC2", 1),
              hdr[:2] + b"\xFF\xCC\x00\x04\x00\x00" + hdr[2:], hdr[:hdr.index(b"\xFF\xDA")] + b"\xFF\xD9"]
    return good, datas


def test_error_isolation(zb, torch):
    good, datas = bad_files(zb)
    fmts = [2] * len(datas)
    status = assert_batch_equals_single(zb, torch, datas, fmts)
    assert status[:len(good)] == [0] * len(good)
    assert {0, 3, 31} <= set(status)
    # a wrong destination shape, a NULL destination and a bad pixel format refuse only their own file
    d0 = good[0]
    h = zb.jpeg_info(d0)
    dsts = [zb.Image.init(h.height, h.width, zb.PixFmt.RGB8) for _ in range(5)]
    dsts[1] = zb.Image.init(h.height, h.width + 1, zb.PixFmt.RGB8)
    for x in dsts:
        x._t.fill_(SENTINEL)
    null = dsts[2]._zb()
    null.data = None
    rc, st, _ = raw_batch(zb, torch, [d0] * 4, [2, 2, 2, 9], dsts=dsts[:4])
    assert rc == 0 and st[0] == 0 and st[1] == 1 and st[3] == 3
    assert (dsts[1]._t == SENTINEL).all() and (dsts[3]._t == SENTINEL).all()
    n = 3
    bufs = [(C.c_uint8 * len(d0)).from_buffer_copy(d0) for _ in range(n)]
    ptrs = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    lens = (C.c_uint64 * n)(*([len(d0)] * n))
    zimg = (zb.ZbImage * n)(dsts[0]._zb(), null, dsts[4]._zb())
    fmt = (C.c_int * n)(2, 2, 2)
    status = (C.c_int * n)()
    assert zb.lib().zb_jpeg_decode_batch(n, ptrs, lens, None, zimg, fmt, status, None) == 0
    assert list(status) == [0, 5, 0]
    want = jd.decode(d0, 2)
    assert np.array_equal(dsts[0].to_numpy(), want) and np.array_equal(dsts[4].to_numpy(), want)


def test_limits_per_file(zb, torch):
    rng = np.random.default_rng(3)
    datas = [jo.encode(content(rng, 20, w, 2), 90, 2) for w in (16, 40, 24)]
    lim = zb.JpegLimits(max_width=30)
    status = assert_batch_equals_single(zb, torch, datas, [2, 2, 2], lim)
    assert status == [0, 30, 0]


def test_two_files_past_2_32_bits(zb, torch):
    rng = np.random.default_rng(8192)
    img = rng.integers(0, 256, (8192, 8192, 3), dtype=np.uint8)
    data = zb.Image.from_numpy(img).encode_jpeg(100, 0)
    del img
    assert 2 * (len(data) - data.index(b"\xFF\xDA")) * 8 > 2 ** 32
    big = zb_limits(zb, BIG)
    want = zb.Image.decode_jpeg(data, 2, big).to_numpy()
    out = zb.Image.decode_jpeg_batch([data, data], 2, big)
    for img in out:
        assert np.array_equal(img.to_numpy(), want)


def test_edges_and_argument_errors(zb, torch):
    L = zb.lib()
    before = L.zb_kernel_launch_count()
    assert L.zb_jpeg_decode_batch(0, None, None, None, None, None, None, None) == 0
    assert L.zb_kernel_launch_count() == before
    d = (FIX / "pillow_optimize_422.jpg").read_bytes()
    h = zb.jpeg_info(d)
    img = zb.Image.init(h.height, h.width, zb.PixFmt.RGBA8)
    buf = (C.c_uint8 * len(d)).from_buffer_copy(d)
    ptrs = (C.c_void_p * 1)(C.addressof(buf))
    lens = (C.c_uint64 * 1)(len(d))
    zimg = (zb.ZbImage * 1)(img._zb())
    fmt = (C.c_int * 1)(3)
    status = (C.c_int * 1)(-1)
    for args in [(None, lens, zimg, fmt, status), (ptrs, None, zimg, fmt, status), (ptrs, lens, None, fmt, status),
                 (ptrs, lens, zimg, None, status), (ptrs, lens, zimg, fmt, None)]:
        a, b, c, e, f = args
        assert L.zb_jpeg_decode_batch(1, a, b, None, c, e, f, None) == 5
    assert status[0] == -1   # rejected before any file was looked at
    assert L.zb_jpeg_decode_batch(1, ptrs, lens, None, zimg, fmt, status, None) == 0 and status[0] == 0
    assert np.array_equal(img.to_numpy(), zb.Image.decode_jpeg(d, 3).to_numpy())
    assert L.zb_last_kernel().decode() == "jpeg_dec_422_rgba8"


def test_streams_and_threads(zb, torch):
    a = mixed_set(zb)
    b = [(FIX / "liza.jpg").read_bytes()] * 8 + a[:5]
    want = {}
    for name, datas in (("a", a), ("b", b)):
        want[name] = [zb.Image.decode_jpeg(d).to_numpy() for d in datas]
    errs = []

    def run(name, datas):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(3):
                    out = zb.Image.decode_jpeg_batch(datas)
                    s.synchronize()
                    for got, w in zip(out, want[name]):
                        assert np.array_equal(got.to_numpy(), w)
        except Exception as e:   # reported below
            errs.append(e)
    ts = [threading.Thread(target=run, args=("a", a)), threading.Thread(target=run, args=("b", b))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_python_mirror(zb, torch):
    good, datas = bad_files(zb)
    gray = jo.encode(content(np.random.default_rng(9), 30, 31, 0), 90)
    datas = [gray] + datas
    out = zb.decode_jpeg_batch(datas)
    assert len(out) == len(datas)
    assert out[0].pixfmt == zb.PixFmt.U8 and out[1].pixfmt == zb.PixFmt.RGB8
    for d, o in zip(datas, out):
        want_rc, want = single(zb, d, None)
        if want_rc:
            assert isinstance(o, zb.ZignalError) and o.status == want_rc
        else:
            assert isinstance(o, zb.Image) and np.array_equal(o.to_numpy(), want)
    fmts = [k % 5 for k in range(len(good))]
    for o, d, f in zip(zb.decode_jpeg_batch(good, fmts), good, fmts):
        assert o.pixfmt == f and np.array_equal(o.to_numpy(), single(zb, d, f)[1])
    assert zb.decode_jpeg_batch([]) == []
