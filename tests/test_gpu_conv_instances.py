"""Every compiled instance of the separable convolution kernels against the oracle.

The kernels are templates on the tap half-width, and the host switches on max(nx / 2, ny / 2) to pick one.  The tests of
test_gpu_conv.py reach the half-widths their tap counts happen to give; this file runs every `case` of every switch, with its
kernel name asserted so that no case can pass on a fallback:
  * fused_sep_rgbaf32[_exact]                 halves 1-8, exact and FFMA arithmetic
  * fused_sep_rgba8_dp / _f / (IMAD)          halves 1-8, the three pipelines of one kernel template (one switch), each
                                              forced with conv.u8_dp / conv.u8_fmath
  * sep_tile_u8[_dp], 1 / 3 / 4 channels      halves 1-15 (dot-product variant 1-8); Rgba through a 3-px view offset
  * conv2d_tile_u8 (dense), 1 / 3 / 4 ch.     halves 1-3
Unequal kx / ky lengths, even tap counts and signed taps, every border mode.  Integer formats and the f32 exact mode must give
the oracle's bits; the f32 FFMA mode is held to a componentwise rounding bound (see _assert_fma_bound).

Two more kinds of coverage the ordinary shapes never reach:
  * fused RGBA f32 and Rgba8 images with more 256-px strips than SMs, so that a persistent CTA runs several work units: stage
    index and mbarrier parity carried from one unit into the next, the next unit's chunks prefetched during the last one, a CTA
    moving from an inner strip to an edge strip.  The shapes are derived from the SM count of the device.
  * Q8 taps on and one step beyond each bound the host proves before it picks an arithmetic path, on images that drive the sums
    to their extremes.

The table INSTANCES is checked against the `case N: return launch_...<N>` lines of the sources without a GPU: adding or
removing an instantiation fails that test until the table, and with it the tests, follow."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

import oracle_lib as zo
from gpu_utils import BORDERS, border_enum

CSRC = Path(__file__).resolve().parent.parent / "zignal_b200" / "csrc"

# (source, launcher) -> the `case` values of its dispatch switch.  The launch_*half* entries are the tile kernels' channel
# switches (4 channels is their `default:` branch); all others are the switches on the tap half-width.
INSTANCES = {
    ("zb_conv_fused.cu", "launch_fused"): list(range(1, 9)),       # fused_sep_rgbaf32, fused_sep_rgbaf32_exact
    ("zb_conv_fused_u8.cu", "launch_u8"): list(range(1, 9)),       # fused_sep_rgba8_dp, fused_sep_rgba8_f (FFMA), fused_sep_rgba8 (IMAD)
    ("zb_conv_tile_u8.cu", "launch_tile_dp"): list(range(1, 9)),   # sep_tile_u8_dp
    ("zb_conv_tile_u8.cu", "launch_tile"): list(range(1, 16)),     # sep_tile_u8
    ("zb_conv_tile_u8.cu", "launch_dense"): list(range(1, 4)),     # conv2d_tile_u8
    ("zb_conv_tile_u8.cu", "launch_half_dp"): [1, 3],
    ("zb_conv_tile_u8.cu", "launch_half"): [1, 3],
    ("zb_conv_tile_u8.cu", "launch_dense_half"): [1, 3],
}
F32_HALVES = INSTANCES[("zb_conv_fused.cu", "launch_fused")]
U8_HALVES = INSTANCES[("zb_conv_fused_u8.cu", "launch_u8")]
TILE_HALVES = INSTANCES[("zb_conv_tile_u8.cu", "launch_tile")]
TILE_DP_HALVES = INSTANCES[("zb_conv_tile_u8.cu", "launch_tile_dp")]
DENSE_HALVES = INSTANCES[("zb_conv_tile_u8.cu", "launch_dense")]
_CASE = re.compile(r"case\s+(\d+)\s*:\s*return\s+(launch_\w+)\s*<\s*(?:CH\s*,\s*)?(\d+)\s*>")


def test_instance_table_matches_dispatch_switches():
    found = {}
    for src in sorted({s for s, _ in INSTANCES}):
        for m in _CASE.finditer((CSRC / src).read_text()):
            case, fn, arg = int(m[1]), m[2], int(m[3])
            assert case == arg, f"{src}: `case {case}` launches {fn}<{arg}>"
            found.setdefault((src, fn), []).append(case)
    assert found == INSTANCES


@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    zo.set_threads(zo.hw_threads())
    yield zb
    L = zb.lib()
    L.zb_set_exact_f32(0)
    L.zb_tune(b"conv.u8_dp", 1)
    L.zb_tune(b"conv.u8_fmath", 1)
    zo.set_threads(1)


def _sm_count(zb):
    n = C.c_int()
    zb._ffi.check(zb.lib().zb_sm_count(C.byref(n)))
    return n.value


# ---- taps -------------------------------------------------------------------------------------------------------------------

def _tap_lengths(half):
    """(nx, ny, signed) tap sets whose max(nx / 2, ny / 2) is `half`: equal odd lengths, an even nx with a shorter ny, an even ny
    with a shorter nx, and signed taps among them."""
    return [(2 * half + 1, 2 * half + 1, False), (2 * half, half, True), (half + 1, 2 * half, False), (2 * half + 1, 2 * half - 1, True)]


def _f32_taps(rng, n, signed):
    """n taps with sum |k| = 1, none of them near the reference's negligible-tap threshold (1e-10); signed: both signs (n >= 2)."""
    while True:
        k = rng.standard_normal(n) if signed else rng.random(n) + 0.05
        k = (k / np.abs(k).sum()).astype(np.float32)
        if np.abs(k).min() > 1e-3 and (not signed or n == 1 or (k.min() < 0 < k.max())):
            return k


def _q8_taps(rng, n, total, signed=False):
    """n Q8 taps, each of magnitude >= 1, whose magnitudes sum to `total`; signed: both signs (n >= 2).  Returned as the integers q
    and the float taps q / 256, which the kernels' roundf(k * 256) maps back to q exactly."""
    assert total >= n >= 1
    w = rng.random(n) + 0.25
    q = np.floor(w / w.sum() * (total - n)).astype(np.int64) + 1
    np.add.at(q, rng.integers(0, n, total - int(q.sum())), 1)
    if signed and n >= 2:
        s = np.where(rng.random(n) < 0.5, -1, 1)
        i, j = rng.choice(n, 2, replace=False)
        s[i], s[j] = -1, 1
        q = q * s
    assert int(np.abs(q).sum()) == total
    return q, (q / 256.0).astype(np.float32)


def _dp_ok(qx, qy):
    """The dot-product pipelines take kernels whose Q8 taps are all bytes and whose horizontal sums fit 16 bits."""
    return bool(qx.min() >= 0 and qx.max() <= 255 and qy.min() >= 0 and qy.max() <= 255 and 255 * int(qx.sum()) <= 65535)


def _fused_u8_kernel(qx, qy, dp, fmath):
    if dp and _dp_ok(qx, qy):
        return "fused_sep_rgba8_dp"
    # exact integers on FFMA: every partial sum is an integer of magnitude <= 255 * sum|kx| * sum|ky| <= 2^24
    if fmath and 255 * int(np.abs(qx).sum()) * int(np.abs(qy).sum()) <= 1 << 24:
        return "fused_sep_rgba8_f"
    return "fused_sep_rgba8"


def _tile_kernel(qx, qy, dp):
    half = max(qx.size // 2, qy.size // 2)
    return "sep_tile_u8_dp" if dp and half <= TILE_DP_HALVES[-1] and _dp_ok(qx, qy) else "sep_tile_u8"


# ---- checks -----------------------------------------------------------------------------------------------------------------

def _assert_fma_bound(got, want, absconv, nx, ny, what):
    """FFMA against the oracle's unfused mul + add: each of the two passes differs by at most n roundings of the partial sums on
    either side, so |got - want| <= 2 (nx + ny) 2^-24 conv(|x|; |kx|, |ky|) + tiny.  A dropped or misplaced tap misses this by
    orders of magnitude, rounding never does.  (The check itself runs in f32: its own rounding is ~2^-24 of the bound.)"""
    bound = np.float32(2 * (nx + ny) * 2.0 ** -24) * absconv
    bound += np.finfo(np.float32).tiny
    err = got - want
    np.abs(err, out=err)
    bad = ~(err <= bound)   # NaN fails too
    if bad.any():
        idx = tuple(int(i[0]) for i in np.nonzero(bad))
        pytest.fail(f"{what}: {int(bad.sum())} values outside the FFMA bound, first at {idx}: got {got[idx]!r} want {want[idx]!r} "
                    f"bound {bound[idx]!r}")


POISON_U8 = 0xA5


def _poisoned(out):
    """Refill `out` (a whole, contiguous Image) with NaN (f32) or 0xA5 (8-bit) and return it.  Every call below writes into a freshly
    poisoned destination, so a pixel a kernel leaves unwritten fails the comparison -- without it, the previous call's identical
    result (or a reused allocation holding it) would stand in for the missing write."""
    t = out.tensor()
    t.fill_(float("nan") if t.is_floating_point() else POISON_U8)
    return out


def _is_poison(a):
    return bool(np.isnan(a).all()) if a.dtype.kind == "f" else bool((a == POISON_U8).all())


def _plateau_u8(rng, shape, qx, qy, band):
    """Random 8-bit image whose first `band` rows tile the pattern that drives the sum of qx (x) qy to its maximum -- 255 where the x
    and the y tap have the same sign, 0 where they differ (all 255 for non-negative taps) -- and whose next `band` rows tile the
    opposite pattern (the minimum)."""
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    hi = np.where(np.sign(qy)[:, None] == np.sign(qx)[None, :], 255, 0).astype(np.uint8)
    cols = shape[1]
    for r0, block in ((0, hi), (band, 255 - hi)):
        t = np.tile(block, (-(-band // block.shape[0]), -(-cols // block.shape[1])))[:band, :cols]
        img[r0:r0 + band] = t[..., None] if img.ndim == 3 else t
    return img


# ---- every half-width, every border mode ------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("half", F32_HALVES)
@pytest.mark.parametrize("rows,cols", [(141, 600), (136, 603)])   # 3 strips (one inner), all four edges; ragged right edge
def test_fused_rgbaf32_every_half(zb, rows, cols, half):
    L = zb.lib()
    rng = np.random.default_rng(1000 * half + cols)
    img = rng.uniform(-1.0, 1.0, (rows, cols, 4)).astype(np.float32)
    dev, out = zb.Image.from_numpy(img), zb.Image.from_numpy(np.empty_like(img))
    for nx, ny, signed in _tap_lengths(half):
        kx, ky = _f32_taps(rng, nx, signed), _f32_taps(rng, ny, signed)
        for border in BORDERS:
            bm = border_enum(zb, border)
            want = zo.conv_separable(img, kx, ky, border)
            absconv = zo.conv_separable(np.abs(img), np.abs(kx), np.abs(ky), border)
            try:
                L.zb_set_exact_f32(1)
                got = dev.convolve_separable(kx, ky, bm, out=_poisoned(out)).to_numpy()
                assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32_exact", (nx, ny, border)
            finally:
                L.zb_set_exact_f32(0)
            assert np.array_equal(got, want), ("exact", nx, ny, border)
            got = dev.convolve_separable(kx, ky, bm, out=_poisoned(out)).to_numpy()
            assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32", (nx, ny, border)
            _assert_fma_bound(got, want, absconv, nx, ny, ("fma", nx, ny, border))


@pytest.mark.gpu
@pytest.mark.parametrize("half", U8_HALVES)
def test_fused_rgba8_every_half_and_pipeline(zb, half):
    L = zb.lib()
    rng = np.random.default_rng(2000 + half)
    img = rng.integers(0, 256, (141, 600, 4), dtype=np.uint8)
    dev, out = zb.Image.from_numpy(img), zb.Image.from_numpy(np.empty_like(img))
    seen = set()
    try:
        for nx, ny, signed in _tap_lengths(half):
            total = 200 if signed else 256     # signed: sum |q| = 200 keeps the FFMA pipeline exact (255 * 200^2 < 2^24)
            (qx, kx), (qy, ky) = _q8_taps(rng, nx, total, signed), _q8_taps(rng, ny, total, signed)
            for border in BORDERS:
                want = zo.conv_separable(img, kx, ky, border)
                for dp, fmath in ((1, 1), (0, 1), (0, 0)):
                    L.zb_tune(b"conv.u8_dp", dp)
                    L.zb_tune(b"conv.u8_fmath", fmath)
                    got = dev.convolve_separable(kx, ky, border_enum(zb, border), out=_poisoned(out)).to_numpy()
                    name = L.zb_last_kernel().decode()
                    assert name == _fused_u8_kernel(qx, qy, dp, fmath), (nx, ny, dp, fmath, name)
                    assert np.array_equal(got, want), (nx, ny, border, name)
                    seen.add(name)
    finally:
        L.zb_tune(b"conv.u8_dp", 1)
        L.zb_tune(b"conv.u8_fmath", 1)
    assert seen == {"fused_sep_rgba8_dp", "fused_sep_rgba8_f", "fused_sep_rgba8"}


# (image shape, view rectangle (l, t, r, b) or None): gray and Rgb rows of 4-byte multiples and odd widths; Rgba through a view 3 px
# (12 bytes) into its buffer, which the 16-byte TMA kernel refuses
TILE_LAYOUTS = {
    "gray_aligned": ((150, 600), None),
    "gray_odd": ((150, 601), None),
    "rgb_aligned": ((150, 400, 3), None),
    "rgb_odd": ((149, 401, 3), None),
    "rgba_view": ((152, 410, 4), (3, 1, 403, 151)),
}


def _layout(zb, rng, name):
    """(source as the oracle sees it, device source, contiguous device destination of the same shape)"""
    shape, rect = TILE_LAYOUTS[name]
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    dev = zb.Image.from_numpy(img)
    if rect is not None:
        l, t, r, b = rect
        img, dev = np.ascontiguousarray(img[t:b, l:r]), dev.view(zb.Rectangle(l, t, r, b))
    return img, dev, zb.Image.from_numpy(np.empty_like(img))


@pytest.mark.gpu
@pytest.mark.parametrize("half", TILE_HALVES)
@pytest.mark.parametrize("layout", list(TILE_LAYOUTS))
def test_tile_u8_every_half(zb, layout, half):
    L = zb.lib()
    rng = np.random.default_rng(3000 + 17 * half + len(layout))
    img, dev, out = _layout(zb, rng, layout)
    seen = set()
    try:
        for nx, ny, signed in _tap_lengths(half):
            (qx, kx), (qy, ky) = _q8_taps(rng, nx, 200 if signed else 256, signed), _q8_taps(rng, ny, 200 if signed else 256, signed)
            for border in BORDERS:
                want = zo.conv_separable(img, kx, ky, border)
                for dp in (1, 0):
                    L.zb_tune(b"conv.u8_dp", dp)
                    got = dev.convolve_separable(kx, ky, border_enum(zb, border), out=_poisoned(out)).to_numpy()
                    name = L.zb_last_kernel().decode()
                    assert name == _tile_kernel(qx, qy, dp), (nx, ny, dp, name)
                    assert np.array_equal(got, want), (nx, ny, border, name)
                    seen.add(name)
    finally:
        L.zb_tune(b"conv.u8_dp", 1)
    assert seen == ({"sep_tile_u8", "sep_tile_u8_dp"} if half in TILE_DP_HALVES else {"sep_tile_u8"})


@pytest.mark.gpu
@pytest.mark.parametrize("half", DENSE_HALVES)
@pytest.mark.parametrize("layout", list(TILE_LAYOUTS))
def test_dense_tile_u8_every_half(zb, layout, half):
    L = zb.lib()
    rng = np.random.default_rng(4000 + half)
    img, dev, out = _layout(zb, rng, layout)
    for kh, kw in [(2 * half + 1, 2 * half + 1), (2 * half, 2 * half - 1), (1, 2 * half)]:
        k = (rng.standard_normal((kh, kw)) / (kh * kw)).astype(np.float32)
        for border in BORDERS:
            got = dev.convolve(k, border_enum(zb, border), out=_poisoned(out)).to_numpy()
            assert L.zb_last_kernel().decode() == "conv2d_tile_u8", (kh, kw)
            assert np.array_equal(got, zo.convolve(img, k, border)), (kh, kw, border)


# ---- several work units per CTA ---------------------------------------------------------------------------------------------

# (rows, cols) from the SM count: one strip more than SMs, short and tall; twice as many strips plus a ragged one (cols % 8 != 0,
# three rounds of strips); a height that is not a multiple of the 8-row chunk
WIDE = {
    "sm+1_strips_64_rows": lambda sm: (64, (sm + 1) * 256),
    "sm+1_strips_1024_rows": lambda sm: (1024, (sm + 1) * 256),
    "2sm+2_strips_ragged": lambda sm: (64, 2 * sm * 256 + 259),
    "rows_not_multiple_of_8": lambda sm: (203, (sm + 1) * 256 + 100),
}
WIDE_HALVES = (1, 5, 8)


def _wide_dst(zb, rows, cols, dtype):
    """A destination buffer 3 rows / 8 px larger on every side and the view of it the convolution writes."""
    big = zb.Image.from_numpy(np.empty((rows + 6, cols + 16, 4), dtype))
    return big, big.view(zb.Rectangle(8, 3, 8 + cols, 3 + rows))


def _wide_result(big, rows, cols, what):
    """The view's pixels after a call into a poisoned `big`; the frame around the view must still be poison."""
    full = big.tensor().cpu().numpy()
    for outside in (full[:3], full[3 + rows:], full[3:3 + rows, :8], full[3:3 + rows, 8 + cols:]):
        assert _is_poison(outside), (what, "pixels outside the destination view were written")
    return full[3:3 + rows, 8:8 + cols]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(WIDE))
def test_fused_rgbaf32_several_units_per_cta(zb, shape):
    """More 256-px strips than SMs: every strip has at least one row segment, so some CTA runs more than one unit."""
    L = zb.lib()
    sm = _sm_count(zb)
    rows, cols = WIDE[shape](sm)
    assert -(-cols // 256) > sm
    rng = np.random.default_rng(rows + cols)
    img = rng.random((rows, cols, 4), dtype=np.float32)
    src = zb.Image.from_numpy(img)
    big, out = _wide_dst(zb, rows, cols, np.float32)
    for half in WIDE_HALVES:
        k = _f32_taps(rng, 2 * half + 1, False)
        for border in BORDERS:
            want = zo.conv_separable(img, k, k, border)   # data and taps >= 0: also conv(|x|; |k|, |k|) of the FFMA bound
            try:
                L.zb_set_exact_f32(1)
                _poisoned(big)
                src.convolve_separable(k, k, border_enum(zb, border), out=out)
                assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32_exact"
            finally:
                L.zb_set_exact_f32(0)
            got = _wide_result(big, rows, cols, ("exact", half, border))
            assert np.array_equal(got, want), ("exact", half, border)
            _poisoned(big)
            src.convolve_separable(k, k, border_enum(zb, border), out=out)
            assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32"
            got = _wide_result(big, rows, cols, ("fma", half, border))
            _assert_fma_bound(got, want, want, k.size, k.size, ("fma", half, border))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(WIDE))
def test_fused_rgba8_several_units_per_cta(zb, shape):
    """The same shapes through the Rgba8 kernel (256-row bands x strips over SMs CTAs, 2 x SMs for the dot-product variant): the
    three pipelines give the oracle's bits.  TMA needs a row pitch of 16-byte multiples, so the source is a view of a buffer whose
    rows are padded to a multiple of 4 pixels (a ragged width of a contiguous image would take the tile kernel)."""
    L = zb.lib()
    sm = _sm_count(zb)
    rows, cols = WIDE[shape](sm)
    assert -(-cols // 256) > sm
    rng = np.random.default_rng(rows * 3 + cols)
    pitch = (cols + 3) // 4 * 4 + 4   # a multiple of 4 px (16-byte rows) that is never cols itself: the source is always a view
    buf = rng.integers(0, 256, (rows, pitch, 4), dtype=np.uint8)
    img = np.ascontiguousarray(buf[:, :cols])
    src = zb.Image.from_numpy(buf).view(zb.Rectangle(0, 0, cols, rows))
    big, out = _wide_dst(zb, rows, cols, np.uint8)
    try:
        for half in WIDE_HALVES:
            qk, k = _q8_taps(rng, 2 * half + 1, 256)
            for border in BORDERS:
                want = zo.conv_separable(img, k, k, border)
                for dp, fmath in ((1, 1), (0, 1), (0, 0)):
                    L.zb_tune(b"conv.u8_dp", dp)
                    L.zb_tune(b"conv.u8_fmath", fmath)
                    _poisoned(big)
                    src.convolve_separable(k, k, border_enum(zb, border), out=out)
                    name = L.zb_last_kernel().decode()
                    assert name == _fused_u8_kernel(qk, qk, dp, fmath), (half, dp, fmath, name)
                    assert np.array_equal(_wide_result(big, rows, cols, (half, border, name)), want), (half, border, name)
    finally:
        L.zb_tune(b"conv.u8_dp", 1)
        L.zb_tune(b"conv.u8_fmath", 1)


# ---- the host's exactness proofs, on and one step beyond their bounds -------------------------------------------------------

def _one_negative(rng, n, total):
    """n Q8 taps with |q| summing to `total`: one of them -1, the rest positive."""
    q, _ = _q8_taps(rng, n - 1, total - 1)
    q = np.insert(q, rng.integers(0, n), -1)
    return q, (q / 256.0).astype(np.float32)


def _run_bound_case(zb, img, dev, qx, kx, qy, ky, expect, what):
    L = zb.lib()
    out = zb.Image.from_numpy(np.empty_like(img))
    for border in BORDERS:
        got = dev.convolve_separable(kx, ky, border_enum(zb, border), out=_poisoned(out)).to_numpy()
        assert L.zb_last_kernel().decode() == expect, (what, border, L.zb_last_kernel().decode())
        assert np.array_equal(got, zo.conv_separable(img, kx, ky, border)), (what, border)


@pytest.mark.gpu
def test_fused_rgba8_ffma_bound(zb):
    """fused_sep_rgba8_f runs the Q8 arithmetic on the FP32 pipe when 255 sum|kx| sum|ky| <= 2^24.  255 does not divide 2^24, so
    the bound's edge is sum|kx| sum|ky| = 65793 (255 x 65793 = 2^24 - 1); 65794 must take the IMAD kernel.  With positive taps the
    all-255 plateau makes the sum exactly 255 sum(kx) sum(ky): 2^24 - 1 on the edge (sum(kx) > 257 keeps the dot-product variant
    out).  The signed pair (one -1 tap per kernel) takes the same decision with the maximum and minimum patterns of mixed signs."""
    rng = np.random.default_rng(51)
    cases = [(273, 241, False, "fused_sep_rgba8_f"), (491, 134, False, "fused_sep_rgba8"),
             (273, 241, True, "fused_sep_rgba8_f"), (134, 491, True, "fused_sep_rgba8")]
    for sx, sy, signed, expect in cases:
        assert (255 * sx * sy <= 1 << 24) == (expect == "fused_sep_rgba8_f")
        if signed:
            (qx, kx), (qy, ky) = _one_negative(rng, 15, sx), _one_negative(rng, 17, sy)
        else:
            (qx, kx), (qy, ky) = _q8_taps(rng, 15, sx), _q8_taps(rng, 17, sy)
        img = _plateau_u8(rng, (96, 600, 4), qx, qy, 34)
        assert _fused_u8_kernel(qx, qy, 1, 1) == expect
        _run_bound_case(zb, img, zb.Image.from_numpy(img), qx, kx, qy, ky, expect, (sx, sy))


# sum(kx) = 255 x 257 = 65535 is the largest horizontal sum a u16 holds; 258 overflows it.  A tap of 255 is a byte, 256 is not.
DP_BOUND_CASES = [
    ("sum_257", lambda rng: _q8_taps(rng, 9, 257), True),
    ("sum_258", lambda rng: _q8_taps(rng, 9, 258), False),
    ("tap_255", lambda rng: (np.array([255, 2]), np.array([255, 2], np.float32) / 256), True),
    ("tap_256", lambda rng: (np.array([256, 1]), np.array([256, 1], np.float32) / 256), False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in DP_BOUND_CASES])
def test_dot_product_bound(zb, case):
    """The dot-product variants (fused Rgba8 and tile) need byte taps and 255 sum(kx) <= 65535: their horizontal sums are u16.  On
    the bound an all-255 plateau makes a horizontal sum of exactly 65535."""
    _, make, dp = next(c for c in DP_BOUND_CASES if c[0] == case)
    rng = np.random.default_rng(61)
    qx, kx = make(rng)
    assert _dp_ok(qx, np.array([0])) == dp
    qy, ky = _q8_taps(rng, 11, 256)
    # fused Rgba8 kernel
    img = _plateau_u8(rng, (96, 600, 4), qx, qy, 34)
    expect = _fused_u8_kernel(qx, qy, 1, 1)
    assert (expect == "fused_sep_rgba8_dp") == dp
    _run_bound_case(zb, img, zb.Image.from_numpy(img), qx, kx, qy, ky, expect, (case, "fused"))
    # tile kernel: gray, Rgb, Rgba through a 3-px view
    for shape in [(96, 600), (96, 400, 3), (96, 404, 4)]:
        full = _plateau_u8(rng, shape, qx, qy, 34)
        dev = zb.Image.from_numpy(full)
        if len(shape) == 3 and shape[2] == 4:
            img, dev = np.ascontiguousarray(full[:, 3:403]), dev.view(zb.Rectangle(3, 0, 403, 96))
        else:
            img = full
        _run_bound_case(zb, img, dev, qx, kx, qy, ky, "sep_tile_u8_dp" if dp else "sep_tile_u8", (case, shape))


@pytest.mark.gpu
def test_tile_dp_no_clamp_bound(zb):
    """sep_tile_u8_dp reads divClampU8(65536) straight from byte 2 of the vertical sum when 255 sum(kx) sum(ky) + 32768 < 2^24.  The
    edge is sum(kx) sum(ky) = 65664 (sum 2^24 - 128 on an all-255 plateau: byte 2 is 255); at 65665 the sum reaches 2^24 + 127, whose
    byte 2 is 0, and the kernel must clamp instead.  Whole 6-row strips, word-aligned rows: the path that reads byte 2."""
    rng = np.random.default_rng(71)
    for sx, sy in ((228, 288), (115, 571)):
        assert (255 * sx * sy + 32768 < 1 << 24) == (sx * sy == 65664)
        qx, kx = _q8_taps(rng, 9, sx)
        qy, ky = _q8_taps(rng, 11, sy)
        assert _tile_kernel(qx, qy, 1) == "sep_tile_u8_dp"
        for shape in [(192, 600), (192, 400, 3)]:
            img = _plateau_u8(rng, shape, qx, qy, 48)
            _run_bound_case(zb, img, zb.Image.from_numpy(img), qx, kx, qy, ky, "sep_tile_u8_dp", (sx, sy, shape))
