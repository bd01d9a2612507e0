"""CPU checks of the JPEG encoder's oracle (oracle/zo_jpeg.cpp) and of the device-free part of zb_jpeg_encode:

- the reference's own round-trip tests (codecs/jpeg.zig:2862-3026) as known answers, decoded with Pillow (libjpeg's IDCT, so the PSNR
  bounds are properties, not exact values);
- an independent numpy restatement of the integer pipeline (rgbToYcbcr, the truncating chroma average, the LLM FDCT vectorised over
  blocks, reciprocal quantisation) against the oracle's per-block coefficients;
- a small baseline Huffman decoder, built from the tables in the file's own DHT, that must recover exactly those coefficients from the
  oracle's entropy-coded segment, the trailing-ZRL rule included (a block whose trailing zero run is a multiple of 16 ends in ZRLs and
  has no EOB);
- header bytes, the stream's tail (entropy data ending on a byte boundary, a padded last byte of 0xFF), the i32 bound of the FDCT, the
  argument errors, status names and zb_jpeg_encode_bound."""
import ctypes as C
import io

import numpy as np
import pytest

import jpeg_oracle as jo
from golden_jpeg import noise, smooth, trailing_runs

QUALITIES = [0, 1, 2, 49, 50, 51, 85, 90, 99, 100, 255]
SIZES = [(1, 1), (1, 13), (13, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33)]

# ---- numpy restatement --------------------------------------------------------------------------------------------------------------

LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51,
                   87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101,
                   72, 92, 95, 98, 112, 100, 103, 99], np.int64)
CHROMA_Q = np.full(64, 99, np.int64)
CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]


def np_tables(quality):
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((base * scale + 50) // 100, 1, 255) for base in (LUMA_Q, CHROMA_Q)]


def np_fdct_pass(v, first):
    """One LLM pass over the last axis (8 values) of an int64 array."""
    c = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
             c2053=16819, c2562=20995, c3072=25172)
    sh = 11 if first else 15

    def ds(x, n):
        return (x + (1 << (n - 1))) >> n

    t0, t7 = v[..., 0] + v[..., 7], v[..., 0] - v[..., 7]
    t1, t6 = v[..., 1] + v[..., 6], v[..., 1] - v[..., 6]
    t2, t5 = v[..., 2] + v[..., 5], v[..., 2] - v[..., 5]
    t3, t4 = v[..., 3] + v[..., 4], v[..., 3] - v[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = np.empty_like(v)
    o[..., 0] = (t10 + t11) * 4 if first else ds(t10 + t11, 2)
    o[..., 4] = (t10 - t11) * 4 if first else ds(t10 - t11, 2)
    z1 = (t12 + t13) * c["c0541"]
    o[..., 2] = ds(z1 + t13 * c["c0765"], sh)
    o[..., 6] = ds(z1 - t12 * c["c1847"], sh)
    z5 = (t4 + t5 + t6 + t7) * c["c1175"]
    za, zb_ = -(t4 + t7) * c["c0899"], -(t5 + t6) * c["c2562"]
    z3, z4 = z5 - (t4 + t6) * c["c1961"], z5 - (t5 + t7) * c["c0390"]
    o[..., 7] = ds(t4 * c["c0298"] + za + z3, sh)
    o[..., 5] = ds(t5 * c["c2053"] + zb_ + z4, sh)
    o[..., 3] = ds(t6 * c["c3072"] + zb_ + z3, sh)
    o[..., 1] = ds(t7 * c["c1501"] + za + z4, sh)
    return o


def np_coefficients(img, quality, subsampling):
    """(n_blocks, 64) quantised coefficients in scan order, natural order inside a block."""
    img = jo.encodable(img)
    rows, cols = img.shape[:2]
    gray = img.ndim == 2
    h, v = (1, 1) if gray or subsampling == 0 else ((2, 1) if subsampling == 1 else (2, 2))
    mh, mw = 8 * v, 8 * h
    pr, pc = -(-rows // mh) * mh, -(-cols // mw) * mw
    src = img[np.minimum(np.arange(pr), rows - 1)][:, np.minimum(np.arange(pc), cols - 1)].astype(np.int64)
    if gray:
        planes = [src]
    else:
        r, g, b = src[..., 0], src[..., 1], src[..., 2]
        planes = [np.clip((19595 * r + 38470 * g + 7471 * b + 32768) >> 16, 0, 255),
                  np.clip(((-11059 * r - 21710 * g + 32768 * b + 32768) >> 16) + 128, 0, 255),
                  np.clip(((32768 * r - 27439 * g - 5329 * b + 32768) >> 16) + 128, 0, 255)]
        planes[1:] = [p.reshape(pr // v, v, pc // h, h).sum(axis=(1, 3)) // (h * v) for p in planes[1:]]
    mr, mc = pr // mh, pc // mw
    y = planes[0].reshape(mr, v, 8, mc, h, 8).transpose(0, 3, 1, 4, 2, 5).reshape(mr * mc, v * h, 64)
    parts = [y]
    for p in planes[1:]:
        parts.append(p.reshape(mr, 8, mc, 8).transpose(0, 2, 1, 3).reshape(mr * mc, 1, 64))
    blocks = np.concatenate(parts, axis=1) - 128
    per = blocks.shape[1]
    ql, qc = np_tables(quality)
    recips = [np.round(2.0 ** 24 / (t.astype(np.float64) * 8.0)).astype(np.int64) for t in (ql, qc)]
    d = np_fdct_pass(blocks.reshape(-1, per, 8, 8), True)
    d = np_fdct_pass(d.transpose(0, 1, 3, 2), False).transpose(0, 1, 3, 2).reshape(-1, per, 64)
    rec = np.stack([recips[0] if k < per - 2 or gray else recips[1] for k in range(per)])
    a = np.abs(d)
    qv = (a * rec + (1 << 23)) >> 24
    return (np.sign(d) * qv).reshape(-1, 64).astype(np.int32)


# ---- baseline decoder ---------------------------------------------------------------------------------------------------------------

def segments(data: bytes):
    """[(marker, payload)] up to SOS, then the entropy-coded bytes (stuffing removed) and what follows them."""
    assert data[:2] == b"\xff\xd8"
    i, segs = 2, []
    while True:
        assert data[i] == 0xFF
        m = data[i + 1]
        ln = int.from_bytes(data[i + 2:i + 4], "big")
        segs.append((m, data[i + 4:i + 2 + ln]))
        i += 2 + ln
        if m == 0xDA:
            break
    end = data.rfind(b"\xff\xd9")
    assert end == len(data) - 2
    raw = data[i:end]
    ent = raw.replace(b"\xff\x00", b"\xff")
    assert ent.count(b"\xff") == raw.count(b"\xff\x00")   # every 0xFF is stuffed, nothing else
    return segs, ent


def huffman_tables(payload: bytes):
    tabs, i = {}, 0
    while i < len(payload):
        tc = payload[i]
        bits = payload[i + 1:i + 17]
        vals = payload[i + 17:i + 17 + sum(bits)]
        code, k, table = 0, 0, {}
        for ln in range(1, 17):
            for _ in range(bits[ln - 1]):
                table[(ln, code)] = vals[k]
                code += 1
                k += 1
            code <<= 1
        tabs[tc] = table
        i += 17 + sum(bits)
    return tabs


def decode(data: bytes):
    """(coefficients (n_blocks, 64) in natural order, per-block list of whether the block ended in EOB, number of padding bits)."""
    segs, ent = segments(data)
    seg = dict(segs)
    tabs = huffman_tables(seg[0xC4])
    sof = seg[0xC0]
    rows, cols, nc = int.from_bytes(sof[1:3], "big"), int.from_bytes(sof[3:5], "big"), sof[5]
    if nc == 1:
        per, layout = 1, [0]
        n_blocks = -(-rows // 8) * -(-cols // 8)
    else:
        h, v = sof[7] >> 4, sof[7] & 15
        per, layout = h * v + 2, [0] * (h * v) + [1, 2]
        n_blocks = -(-rows // (8 * v)) * -(-cols // (8 * h)) * per
    bits = np.unpackbits(np.frombuffer(ent, np.uint8))
    pos = 0

    def read(n):
        nonlocal pos
        v_ = 0
        for _ in range(n):
            v_ = (v_ << 1) | int(bits[pos])
            pos += 1
        return v_

    def symbol(table):
        code = 0
        for ln in range(1, 17):
            code = (code << 1) | read(1)
            if (ln, code) in table:
                return table[(ln, code)]
        raise AssertionError("invalid Huffman code")

    def extend(v_, s):
        return v_ - (1 << s) + 1 if s and v_ < (1 << (s - 1)) else v_

    out = np.zeros((n_blocks, 64), np.int32)
    eob = []
    prev = [0, 0, 0]
    for b in range(n_blocks):
        comp = layout[b % per]
        dct, act = tabs[0x00 | (comp > 0)], tabs[0x10 | (comp > 0)]
        s = symbol(dct)
        prev[comp] += extend(read(s), s)
        out[b, 0] = prev[comp]
        k, ended = 1, False
        while k < 64:
            rs = symbol(act)
            r, s = rs >> 4, rs & 15
            if rs == 0x00:
                ended = True
                break
            if rs == 0xF0:
                k += 16
                continue
            k += r
            out[b, jo.ZIGZAG[k]] = extend(read(s), s)
            k += 1
        assert k <= 64
        eob.append(ended)
    pad = len(bits) - pos
    assert pad < 8 and all(bits[pos:])   # flush pads with 1-bits
    return out, eob, pad


# ---- tests --------------------------------------------------------------------------------------------------------------------------

def _psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def _kat_rgb(rows, cols, blue):
    y, x = np.mgrid[0:rows, 0:cols]
    return np.stack([(x * 255) // (cols - 1), (y * 255) // (rows - 1), blue(x, y)], -1).astype(np.uint8)


KATS = [  # (image, quality, subsampling, bound): jpeg.zig:2862-3026
    # Pillow misses this bound (38.5 dB): libjpeg rebuilds 4:2:0 chroma with its triangular "fancy" upsampler, while zignal's decoder
    # interpolates bilinearly (jpeg.zig:2693-2700), and on a 16 x 16 gradient the 8 x 8 chroma plane is all edge.  The same bytes at
    # 4:4:4 give 45 dB, and the coefficient and decoder tests below pin the bytes themselves.
    pytest.param("16x16 rgb", lambda: _kat_rgb(16, 16, lambda x, y: ((x + y) * 255) // 30), 85, 2, 40.0,
                 marks=pytest.mark.xfail(strict=True, reason="libjpeg's fancy chroma upsampling, not zignal's decoder")),
    ("16x16 gray", lambda: ((np.add.outer(np.arange(16), np.arange(16)) * 255) // 30).astype(np.uint8), 85, 2, 45.0),
    ("19x25 422", lambda: _kat_rgb(19, 25, lambda x, y: ((x * y) * 255) // (24 * 18)), 85, 1, 40.0),
    ("64x48 420", lambda: _kat_rgb(64, 48, lambda x, y: ((x + 2 * y) * 255) // (47 + 2 * 63)), 92, 2, 45.0),
    ("37x53 420", lambda: _kat_rgb(37, 53, lambda x, y: ((2 * x + 3 * y) * 255) // (2 * 52 + 3 * 36)), 85, 2, 35.0),
]


@pytest.mark.parametrize("name,make,quality,sub,bound", KATS, ids=["16x16 rgb", "16x16 gray", "19x25 422", "64x48 420", "37x53 420"])
def test_reference_roundtrip_psnr(name, make, quality, sub, bound):
    Image = pytest.importorskip("PIL.Image")
    img = make()
    data = jo.encode(img, quality, sub)
    dec = np.asarray(Image.open(io.BytesIO(data)))
    assert dec.shape == img.shape
    assert _psnr(img, dec) > bound


@pytest.mark.parametrize("kind", ["gray", 0, 1, 2])
@pytest.mark.parametrize("quality", QUALITIES)
def test_numpy_restatement_and_decoder_agree_with_oracle(kind, quality):
    for k, (rows, cols) in enumerate(SIZES):
        img = (smooth("u8", rows, cols, k) if kind == "gray" else smooth("rgb8", rows, cols, k)) if k % 2 else \
            (noise("u8", rows, cols, k) if kind == "gray" else noise("rgb8", rows, cols, k))
        sub = 0 if kind == "gray" else kind
        want = jo.coefficients(img, quality, sub)
        assert np.array_equal(np_coefficients(img, quality, sub), want), (rows, cols)
        got, _, _ = decode(jo.encode(img, quality, sub))
        assert np.array_equal(got, want), (rows, cols)


@pytest.mark.parametrize("fmt", ["f32", "rgba8", "rgbaf32"])
def test_other_formats_encode_as_rgb(fmt):
    img = smooth(fmt, 21, 35, 3)
    assert jo.encode(img, 90, 1) == jo.encode(jo.encodable(img), 90, 1)
    assert np.array_equal(np_coefficients(img, 90, 1), jo.coefficients(img, 90, 1))


def test_trailing_zero_runs_end_in_zrl_without_eob():
    img = trailing_runs(128, 128, 9)
    coefs = jo.coefficients(img, 50, 0)
    got, eob, _ = decode(jo.encode(img, 50, 0))
    assert np.array_equal(got, coefs)
    zz = coefs[:, jo.ZIGZAG]
    last = np.array([np.nonzero(r[1:])[0].max() + 1 if np.any(r[1:]) else 0 for r in zz])
    for run in (16, 32, 48):
        sel = np.nonzero(63 - last == run)[0]
        assert sel.size, run
        assert not any(eob[i] for i in sel), run
    assert all(eob[i] for i in np.nonzero((63 - last) % 16 != 0)[0])


def test_header_segments():
    img = smooth("rgb8", 20, 30, 1)
    for comment in (None, b"", b"c" * 65533):
        data = jo.encode(img, 75, 1, 300, comment)
        segs, _ = segments(data)
        markers = [m for m, _ in segs]
        assert markers == [0xE0] + ([0xFE] if comment is not None else []) + [0xDB, 0xC0, 0xC4, 0xDA]
        seg = dict(segs)
        assert seg[0xE0] == b"JFIF\x00\x01\x01\x01" + (300).to_bytes(2, "big") * 2 + b"\x00\x00"
        if comment is not None:
            assert seg[0xFE] == comment
        ql, qc = np_tables(75)
        assert seg[0xDB] == bytes([0]) + bytes(ql[jo.ZIGZAG].tolist()) + bytes([1]) + bytes(qc[jo.ZIGZAG].tolist())
        assert seg[0xC0] == bytes([8, 0, 20, 0, 30, 3, 1, 0x21, 0, 2, 0x11, 1, 3, 0x11, 1])
        assert len(seg[0xC4]) == 2 * (17 + 12) + 2 * (17 + 162)
        assert seg[0xDA] == bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    gray = jo.encode(smooth("u8", 9, 11, 2), 90, 2)
    seg = dict(segments(gray)[0])
    assert len(seg[0xDB]) == 65 and seg[0xC0][5:] == bytes([1, 1, 0x11, 0]) and len(seg[0xC4]) == 17 + 12 + 17 + 162
    assert seg[0xDA] == bytes([1, 1, 0, 0, 63, 0])
    with pytest.raises(jo.OracleStatus):
        jo.encode(img, comment=b"c" * 65534)


# Seeds of u8 noise images, 8 x 8 at quality 90, found by search: the entropy data of the first ends exactly on a byte boundary (no
# padding), the padded last byte of the second is 0xFF (so the padding itself is stuffed).
TAIL_ALIGNED_SEED = 1
TAIL_FF_SEED = 10


def _tail(seed):
    data = jo.encode(noise("u8", 8, 8, seed), 90, 0)
    _, _, pad = decode(data)
    return data, pad


def test_stream_tail_cases():
    data, pad = _tail(TAIL_ALIGNED_SEED)
    assert pad == 0
    data, pad = _tail(TAIL_FF_SEED)
    assert pad > 0 and data[-4:] == b"\xff\x00\xff\xd9"


def test_fdct_i32_bound():
    """Propagate intervals through both passes of the LLM FDCT for samples in [-128, 127]: every intermediate of pass 2 stays below
    3.2e8 < 2^31 / 6, so the device's i32 arithmetic gives the reference's i64 results."""
    # each quantity is a linear form over the 8 inputs of its pass; its range is sum |coef| * max |input|
    eye = [np.eye(8, dtype=np.int64)[k] for k in range(8)]

    def forms(x):
        c = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
                 c2053=16819, c2562=20995, c3072=25172)
        t0, t7, t1, t6 = x[0] + x[7], x[0] - x[7], x[1] + x[6], x[1] - x[6]
        t2, t5, t3, t4 = x[2] + x[5], x[2] - x[5], x[3] + x[4], x[3] - x[4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        z1 = (t12 + t13) * c["c0541"]
        z5 = (t4 + t5 + t6 + t7) * c["c1175"]
        za, zb_ = -(t4 + t7) * c["c0899"], -(t5 + t6) * c["c2562"]
        z3, z4 = z5 - (t4 + t6) * c["c1961"], z5 - (t5 + t7) * c["c0390"]
        outs = {0: t10 + t11, 4: t10 - t11, 2: z1 + t13 * c["c0765"], 6: z1 - t12 * c["c1847"], 7: t4 * c["c0298"] + za + z3,
                5: t5 * c["c2053"] + zb_ + z4, 3: t6 * c["c3072"] + zb_ + z3, 1: t7 * c["c1501"] + za + z4}
        inter = [t0, t7, t1, t6, t2, t5, t3, t4, t10, t13, t11, t12, z1, z5, za, zb_, z3, z4, t4 * c["c0298"], t5 * c["c2053"],
                 t6 * c["c3072"], t7 * c["c1501"], t13 * c["c0765"], t12 * c["c1847"], z1 + t13 * c["c0765"]]
        return outs, inter + list(outs.values())

    o1, i1 = forms(eye)
    pass1_max = max(int(np.abs(f).sum()) * 128 for f in i1)
    # pass-1 outputs: 0 and 4 are scaled by 4; the others descaled by 2^11 (rounding adds at most 1)
    r1 = np.array([int(np.abs(o1[k]).sum()) * 128 * 4 if k in (0, 4) else int(np.abs(o1[k]).sum()) * 128 // 2 ** 11 + 1
                   for k in range(8)], np.int64)
    _, i2 = forms(eye)
    pass2_max = max(int((np.abs(f) * r1).sum()) for f in i2)
    assert pass1_max < 2 ** 31 and pass2_max < 3.2e8 < 2 ** 31 / 6


def test_argument_errors_and_status_names():
    import zignal_b200 as zb
    L = zb.lib()
    assert L.zb_status_name(29).decode() == "InvalidImageDimensions" and L.zb_status_name(30).decode() == "ImageTooLarge"
    opts = zb._ffi.ZbJpegOptions(90, 2, 72, None, 0)
    n = C.c_uint64(0)
    img = zb.ZbImage(C.c_void_p(16), 8, 8, 8)   # never dereferenced: every case fails before any device work
    assert L.zb_jpeg_encode(None, 2, C.byref(opts), None, 0, C.byref(n), None) == 5
    assert L.zb_jpeg_encode(C.byref(img), 2, None, None, 0, C.byref(n), None) == 5
    assert L.zb_jpeg_encode(C.byref(img), 2, C.byref(opts), None, 0, None, None) == 5
    assert L.zb_jpeg_encode(C.byref(img), 9, C.byref(opts), None, 0, C.byref(n), None) == 3
    for rows, cols, want in ((0, 8, 29), (8, 0, 29), (65536, 8, 30), (8, 65536, 30)):
        bad = zb.ZbImage(C.c_void_p(16), rows, cols, max(cols, 1))
        assert L.zb_jpeg_encode(C.byref(bad), 2, C.byref(opts), None, 0, C.byref(n), None) == want
        assert L.zb_jpeg_encode_bound(rows, cols, 2, C.byref(opts), C.byref(n)) == want
    for bad_opts in (zb._ffi.ZbJpegOptions(90, 3, 72, None, 0), zb._ffi.ZbJpegOptions(90, 2, 72, C.c_void_p(16), 65534)):
        assert L.zb_jpeg_encode(C.byref(img), 2, C.byref(bad_opts), None, 0, C.byref(n), None) == 5
        assert L.zb_jpeg_encode_bound(8, 8, 2, C.byref(bad_opts), C.byref(n)) == 5
    assert L.zb_jpeg_encode(C.byref(img), 2, C.byref(opts), None, 10, C.byref(n), None) == 5   # NULL out with a capacity


@pytest.mark.parametrize("fmt,sub", [("rgb8", 0), ("rgb8", 2), ("u8", 0)])
def test_bound_covers_noise_at_q100(fmt, sub):
    import zignal_b200 as zb
    for rows, cols in ((1, 1), (8, 8), (37, 53), (128, 96)):
        img = noise(fmt, rows, cols, rows + cols)
        want = len(jo.encode(img, 100, sub, 72, b"x" * 100))
        assert zb.jpeg_encode_bound(rows, cols, zb.PixFmt.RGB8 if fmt == "rgb8" else zb.PixFmt.U8, 100, sub, 72, b"x" * 100) >= want
