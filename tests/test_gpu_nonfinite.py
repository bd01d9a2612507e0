"""Every float entry point with NaN, infinities, signed zeros, subnormals and values outside [0, 1], against the oracle.

One generator (`planted`) writes special values into an otherwise random image: isolated interior pixels, every edge and corner
(so that replicate, mirror and wrap carry them), one whole row, and four consecutive 16-byte-aligned pixels for the vectorised
loaders.  Results are compared bit for bit (`assert_same_bits`): the NaN masks must be identical, any NaN matches any NaN (a NaN's
payload and sign are not pinned, DESIGN.md §7), and the sign of every infinity and every zero must match.  The FFMA fused
convolution keeps the same non-finite masks and Inf signs; its finite values are held to the bound of `_assert_fma_bound`.

Float -> 8-bit conversions clamp with the reference's std.math.clamp(v, 0, 1), whose @min / @max return the non-NaN operand: NaN
gives 255 (tests/test_clamp_rule.py checks the oracle against hand-derived values).

FLOAT_ENTRY_POINTS classifies every `zb_*` entry point of include/zignal_b200.h that takes a pixel format; a CPU test fails when
the header gains one the table does not classify, and a GPU test checks that the 8-bit-only ones refuse an F32 image."""
import ctypes as C
import math
import re
from pathlib import Path

import numpy as np
import pytest

import oracle_lib as zo
import quantize_oracle as qo
import shen_castan_oracle as sco
from gpu_utils import BORDERS, METHODS, border_enum, method_enum

HEADER = Path(__file__).resolve().parent.parent / "include" / "zignal_b200.h"

# Every zb_* function of the header with a pixel-format parameter.  "float": accepts F32 and / or RGBAF32 and is run here with
# special values.  "float, same kernel as X": runs the kernels of X, which is run here.  "float, no arithmetic": accepts float images
# but only moves or compares their bits (or writes a constant), so special values cannot take another path.  "float, elsewhere":
# special values are tested in the named file.  "8-bit only":
# refuses F32 with Unsupported (test_eight_bit_entry_points_refuse_f32).
FLOAT_ENTRY_POINTS = {
    "zb_set_border_zero": "float, no arithmetic",
    "zb_upload": "float, no arithmetic",
    "zb_download": "float, no arithmetic",
    "zb_copy": "float, no arithmetic",
    "zb_conv_separable": "float",
    "zb_conv_separable_rows": "float, same kernel as zb_conv_separable",
    "zb_convolve": "float",
    "zb_gaussian_blur": "float",
    "zb_box_blur": "float",
    "zb_sharpen": "float",
    "zb_integral_plane": "float, same kernel as zb_box_blur",
    "zb_resize": "float",
    "zb_rotate_into": "float",
    "zb_rotate_into_cs": "float",
    "zb_rotate_into_batch": "float, same kernel as zb_rotate_into_cs",
    "zb_warp": "float",
    "zb_sobel": "float",
    "zb_canny": "float",
    "zb_shen_castan": "float",
    "zb_order_blur": "8-bit only",
    "zb_motion_blur_linear": "float",
    "zb_motion_blur_radial": "float",
    "zb_histogram": "8-bit only",
    "zb_autocontrast": "8-bit only",
    "zb_equalize": "8-bit only",
    "zb_flood_fill": "float, elsewhere: test_gpu_flood_fill.py",
    "zb_median_cut": "float",
    "zb_build_palette": "float",                    # zb_median_cut for the adaptive mode
    "zb_dither": "8-bit only",
    "zb_palette_lookup": "float",
    "zb_convert": "float",
    "zb_psnr": "float",
    "zb_ssim": "float",
    "zb_mean_pixel_error": "float",
    "zb_diff": "float, elsewhere: test_gpu_visual.py",
    "zb_apply_colormap": "float, elsewhere: test_gpu_visual.py",
    "zb_flip_left_right": "float, no arithmetic",
    "zb_flip_top_bottom": "float, no arithmetic",
    "zb_invert": "float, elsewhere: test_gpu_visual.py",
    "zb_extract": "float",
    "zb_insert": "float, same kernel as zb_insert_from",
    "zb_insert_blend": "float, same kernel as zb_insert_from",
    "zb_insert_from": "float",
    "zb_jpeg_encode_bound": "float, no arithmetic",  # a byte count from the shape
    "zb_jpeg_encode": "float",
    "zb_jpeg_decode": "float, no arithmetic",        # float destinations receive u8 / 255
    "zb_jpeg_decode_batch": "float, no arithmetic",
    "zb_fdm_create": "8-bit only",
    "zb_fdm_moments": "8-bit only",
    "zb_shard_image_create": "float, no arithmetic",   # describes a row block; the sharded filters are the single-GPU kernels
    "zb_host_conv_separable": "float",
    "zb_host_convolve": "float",
    "zb_host_gaussian_blur": "float",
    "zb_host_box_blur": "float",
    "zb_host_sharpen": "float",
    "zb_host_resize": "float",
    "zb_host_rotate_into": "float",
    "zb_host_warp": "float",
    "zb_host_fdm_match": "8-bit only",
}
CLASSES = {"float", "float, no arithmetic", "8-bit only"}


def _header_pixfmt_functions():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return {m[1] for m in re.finditer(r"\b(zb_\w+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S) if "pixfmt" in m[2]}


def test_entry_point_table_matches_header():
    found = _header_pixfmt_functions()
    assert found == set(FLOAT_ENTRY_POINTS), (sorted(found - set(FLOAT_ENTRY_POINTS)), sorted(set(FLOAT_ENTRY_POINTS) - found))
    for name, cls in FLOAT_ENTRY_POINTS.items():
        assert cls in CLASSES or cls.startswith(("float, elsewhere: ", "float, same kernel as ")), (name, cls)
        if cls.startswith("float, elsewhere: "):
            assert (HEADER.parent.parent / "tests" / cls.split(": ")[1]).exists(), (name, cls)
        if cls.startswith("float, same kernel as "):
            assert FLOAT_ENTRY_POINTS[cls.split(" as ")[1]] == "float", (name, cls)


# ---- special values -----------------------------------------------------------------------------------------------------------

F32 = np.float32
FMAX = np.finfo(F32).max
NAN_POS = np.array([0x7FC00000], np.uint32).view(F32)[0]
NAN_NEG = np.array([0xFFC00000], np.uint32).view(F32)[0]
SUBNORMAL = np.nextafter(F32(0), F32(1))
SPECIAL = np.array([NAN_POS, NAN_NEG, np.inf, -np.inf, 0.0, -0.0, SUBNORMAL, FMAX, -FMAX, 1e30, np.nextafter(F32(1), F32(2)),
                    -SUBNORMAL] + [(k + 0.5) / 255 for k in (0, 1, 127, 254)], F32)
# no +-FLT_MAX / 1e30: sums of such values may round to +-Inf on one side of an FMA and not on the other
SPECIAL_NO_HUGE = SPECIAL[np.isnan(SPECIAL) | (np.abs(SPECIAL) < 1e29) | np.isinf(SPECIAL)]


def planted(rng, shape, values=SPECIAL, rows_full=True):
    """A random [0, 1) image of `shape` ((rows, cols) or (rows, cols, 4)) with `values` planted, cycling, at: isolated interior pixels,
    the four corners and pixels along every edge, one whole row (rows_full) and four consecutive 16-byte-aligned pixels.  Colour
    images get a different value in every channel, plus one pixel whose colour channels are all -0 and one all -subnormal."""
    img = rng.random(shape, dtype=F32)
    rows, cols = shape[:2]
    ch = shape[2] if len(shape) == 3 else 1
    pos = []
    for r in range(3, rows - 3, 7):                                     # isolated interior pixels
        for c in range(3 + (r % 5), cols - 3, 11):
            pos.append((r, c))
    pos += [(0, 0), (0, cols - 1), (rows - 1, 0), (rows - 1, cols - 1)]   # corners
    for t in range(2, cols - 2, max(3, cols // 9)):                       # edges
        pos += [(0, t), (rows - 1, t)]
    for t in range(2, rows - 2, max(3, rows // 9)):
        pos += [(t, 0), (t, cols - 1)]
    if rows_full:
        pos += [(rows // 2 + 1, c) for c in range(cols)]
    flat0 = ((rows // 3) * cols + cols // 2 + 3) // 4 * 4               # 4 consecutive pixels at a 16-byte offset of the plane
    pos += [divmod(flat0 + k, cols) for k in range(4)]
    k = 0
    for r, c in pos:
        if ch == 1:
            img[r, c] = values[k % len(values)]
        else:
            img[r, c] = [values[(k + j * 5) % len(values)] for j in range(ch)]
        k += 1
    if ch == 4:                                                         # colours whose luma is -0 or a negative subnormal
        img[1, 2, :3] = -0.0
        img[2, 1, :3] = -SUBNORMAL
    return img


def _canon(a):
    u = np.ascontiguousarray(a).view(np.uint32).copy()
    u[np.isnan(a)] = 0x7FC00000
    return u


def assert_same_bits(got, want, what=""):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    if got.dtype != np.float32:
        if not np.array_equal(got, want):
            idx = tuple(int(i[0]) for i in np.nonzero(got != want))
            pytest.fail(f"{what}: {int((got != want).sum())} values differ, first at {idx}: got {got[idx]!r} want {want[idx]!r}")
        return
    gn, wn = np.isnan(got), np.isnan(want)
    if not np.array_equal(gn, wn):
        idx = tuple(int(i[0]) for i in np.nonzero(gn != wn))
        pytest.fail(f"{what}: NaN masks differ ({int((gn != wn).sum())}), first at {idx}: got {got[idx]!r} want {want[idx]!r}")
    cg, cw = _canon(got), _canon(want)
    if not np.array_equal(cg, cw):
        idx = tuple(int(i[0]) for i in np.nonzero(cg != cw))
        pytest.fail(f"{what}: {int((cg != cw).sum())} values differ, first at {idx}: got {got[idx]!r} want {want[idx]!r}")


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


def assert_fma_close(got, want, absconv, nx, ny, what):
    """Identical non-finite masks, the same Inf signs, and finite values within the FFMA bound."""
    gf, wf = np.isfinite(got), np.isfinite(want)
    assert np.array_equal(gf, wf), (what, "non-finite masks differ", int((gf != wf).sum()))
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, "NaN masks differ")
    inf = np.isinf(want)
    assert np.array_equal(np.signbit(got[inf]), np.signbit(want[inf])), (what, "Inf signs differ")
    with np.errstate(invalid="ignore", over="ignore"):
        _assert_fma_bound(np.where(wf, got, 0).astype(F32), np.where(wf, want, 0).astype(F32), np.where(wf, absconv, 0).astype(F32),
                          nx, ny, what)


# ---- fixtures -------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    yield zb
    L = zb.lib()
    L.zb_set_exact_f32(0)
    L.zb_set_force_generic(0)
    L.zb_tune(b"conv.edge_fast", 1)


def _kernel(zb):
    return zb.lib().zb_last_kernel().decode()


FLOAT_SHAPES = {"f32": (37, 53), "rgbaf32": (37, 53, 4)}
SENTINEL = F32(-123.5)


def _oracle_quiet():
    return np.errstate(invalid="ignore", over="ignore", divide="ignore")


# ---- convert and mixed insert ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("src", list(FLOAT_SHAPES))
@pytest.mark.parametrize("dst", range(5))
def test_convert(zb, src, dst):
    img = planted(np.random.default_rng(11 + dst), FLOAT_SHAPES[src])
    got = zb.Image.from_numpy(img).convert(zb.PixFmt(dst)).to_numpy()
    if zo.pixfmt_of(img) != dst:
        assert _kernel(zb) == "convert"
    assert_same_bits(got, zo.convert(img, dst), (src, dst))


def _oracle_insert_mixed(dest, source, rect, angle, method):
    """Image.insert of a float source into a destination of another pixel type, from oracle pieces: the sample each destination
    pixel receives is what the same-type insert writes (two canvases with different bits tell written pixels from untouched ones;
    bit equality, so that a NaN sample counts as written), then convertColor(DestType, sample)."""
    shape = dest.shape[:2] + tuple(source.shape[2:])
    s0 = zo.insert(np.zeros(shape, source.dtype), source, rect, angle, method)
    s1 = zo.insert(np.ones(shape, source.dtype), source, rect, angle, method)
    same = s0.view(np.uint32) == s1.view(np.uint32)
    written = same if same.ndim == 2 else same.all(axis=2)
    out = dest.copy()
    conv = zo.convert(s0, zo.pixfmt_of(dest)) if zo.pixfmt_of(dest) != zo.pixfmt_of(source) else s0
    out[written] = conv[written]
    return out


_MIX = {0: ((), np.uint8), 1: ((), np.float32), 2: ((3,), np.uint8), 3: ((4,), np.uint8), 4: ((4,), np.float32)}


@pytest.mark.gpu
@pytest.mark.parametrize("src", list(FLOAT_SHAPES))
@pytest.mark.parametrize("dst", range(5))
def test_insert_from_another_type(zb, src, dst):
    rng = np.random.default_rng(21 + dst)
    source = planted(rng, (24, 30) + FLOAT_SHAPES[src][2:])
    if zo.pixfmt_of(source) == dst:
        pytest.skip("same pixel type: test_insert_and_extract")
    tail, dt = _MIX[dst]
    dest = (rng.integers(0, 256, (40, 52) + tail, dtype=np.uint8) if dt == np.uint8 else rng.random((40, 52) + tail, dtype=F32))
    for rect, angle, method in [((6.0, 5.0, 41.0, 33.0), 0.35, "bilinear"), ((10.0, 8.0, 40.0, 32.0), 0.0, "nearest"),
                                ((3.5, 2.0, 30.0, 38.0), -1.1, "bicubic")]:
        d = zb.Image.from_numpy(dest)
        d.insert(zb.Image.from_numpy(source), rect, angle, method_enum(zb, method))
        assert _kernel(zb) == "insert_mixed"
        with _oracle_quiet():
            want = _oracle_insert_mixed(dest, source, rect, angle, method)
        assert_same_bits(d.to_numpy(), want, (src, dst, rect, method))


# ---- convolution -----------------------------------------------------------------------------------------------------------------

def _taps(rng, n, total=1.0):
    k = rng.random(n) + 0.05
    return (k / k.sum() * total).astype(F32)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_convolve_separable_generic(zb, fmt):
    """The two-pass kernel: F32 always, RGBAF32 when the fused kernel is switched off."""
    rng = np.random.default_rng(31)
    img = planted(rng, FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    L = zb.lib()
    try:
        L.zb_set_force_generic(1)
        for nx, ny in ((5, 5), (4, 7), (1, 9)):
            kx, ky = _taps(rng, nx), _taps(rng, ny)
            kx[0] = -kx[0]
            for border in BORDERS:
                got = dev.convolve_separable(kx, ky, border_enum(zb, border)).to_numpy()
                assert _kernel(zb) == "sep_generic_f32", (nx, ny, border)
                with _oracle_quiet():
                    want = zo.conv_separable(img, kx, ky, border)
                assert_same_bits(got, want, (fmt, nx, ny, border))
    finally:
        L.zb_set_force_generic(0)


@pytest.mark.gpu
@pytest.mark.parametrize("edge_fast", [1, 0])
def test_convolve_separable_fused_rgbaf32(zb, edge_fast):
    """The fused TMA kernel, exact and FFMA arithmetic, with the 8-column x-border copies on (replicate / mirror, cols % 8 == 0) and
    off.  Taps summing to 1/2 keep every finite sum far from FLT_MAX on both sides of an FMA.  Unequal and even lengths pad the
    shorter kernel to 2 * half + 1 taps, which the kernel must skip, not multiply."""
    rng = np.random.default_rng(41 + edge_fast)
    img = planted(rng, (96, 520, 4), SPECIAL_NO_HUGE)
    dev = zb.Image.from_numpy(img)
    L = zb.lib()
    try:
        L.zb_tune(b"conv.edge_fast", edge_fast)
        for nx, ny in ((15, 15), (7, 7), (3, 8), (4, 4), (1, 9), (9, 2)):
            kx, ky = _taps(rng, nx, 0.5), _taps(rng, ny, 0.5)
            ky[1] = -ky[1]
            for border in BORDERS:
                with _oracle_quiet():
                    want = zo.conv_separable(img, kx, ky, border)
                    absconv = zo.conv_separable(np.abs(img), np.abs(kx), np.abs(ky), border)
                try:
                    L.zb_set_exact_f32(1)
                    got = dev.convolve_separable(kx, ky, border_enum(zb, border)).to_numpy()
                    assert _kernel(zb) == "fused_sep_rgbaf32_exact"
                finally:
                    L.zb_set_exact_f32(0)
                assert_same_bits(got, want, ("exact", nx, ny, border))
                got = dev.convolve_separable(kx, ky, border_enum(zb, border)).to_numpy()
                assert _kernel(zb) == "fused_sep_rgbaf32"
                assert_fma_close(got, want, absconv, nx, ny, ("fma", nx, ny, border))
    finally:
        L.zb_tune(b"conv.edge_fast", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [1, 0])
def test_fused_padded_taps_meet_nonfinite(zb, exact):
    """kx = [1, 2, 1] / 4, ky = [1]: the fused kernel pads ky to three taps.  A NaN and an Inf pixel must spread along their row only
    (the columns of kx's support), never into the rows above and below, which the padding taps would reach.  Hand-derived masks,
    then the oracle."""
    rng = np.random.default_rng(45)
    img = rng.random((96, 520, 4), dtype=F32)
    img[40, 100] = np.nan
    img[60, 200] = np.inf
    kx, ky = np.array([0.25, 0.5, 0.25], F32), np.ones(1, F32)
    nan_mask = np.zeros(img.shape, bool)
    nan_mask[40, 99:102] = True
    inf_mask = np.zeros(img.shape, bool)
    inf_mask[60, 199:202] = True
    L = zb.lib()
    for border in BORDERS:
        try:
            L.zb_set_exact_f32(exact)
            got = zb.Image.from_numpy(img).convolve_separable(kx, ky, border_enum(zb, border)).to_numpy()
            assert _kernel(zb) == ("fused_sep_rgbaf32_exact" if exact else "fused_sep_rgbaf32")
        finally:
            L.zb_set_exact_f32(0)
        assert np.array_equal(np.isnan(got), nan_mask), (border, int(np.isnan(got).sum()))
        assert np.array_equal(np.isposinf(got), inf_mask) and not np.isneginf(got).any(), border
        with _oracle_quiet():
            want = zo.conv_separable(img, kx, ky, border)
        if exact:
            assert_same_bits(got, want, ("padded taps", border))
        else:
            assert_fma_close(got, want, zo.conv_separable(np.abs(img), kx, ky, border), 3, 1, ("padded taps", border))


def _zero_tap_expected(img, axis):
    """Hand derivation of the 3-tap (1/2, 0, 1/2) convolution along `axis` (the other kernel is [1]) for one Inf pixel at index 10 of
    that axis and one at index 0: the reference skips |k| < 1e-10 in the interior only (convolution.zig:459-467, 537-548), so the
    interior neighbours of an Inf pixel are Inf, the Inf pixel itself gets 0.5 x[i-1] + 0.5 x[i+1], and the border pixel index 0
    gets 0 * Inf = NaN.  Returns (pixel -> expected value) for those pixels of line 5 of the other axis."""
    line = img[5] if axis == 1 else img[:, 5]
    h = lambda v: (F32(0.5) * np.asarray(v, F32)).astype(F32)                  # noqa: E731
    inner = ((F32(0) + h(line[9])).astype(F32) + h(line[11])).astype(F32)
    inf, nan = np.full_like(inner, np.inf), np.full_like(inner, np.nan)
    return {9: inf, 10: inner, 11: inf, 0: nan, 1: inf}


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
@pytest.mark.parametrize("axis", [1, 0])
def test_zero_tap_meets_inf(zb, fmt, axis):
    """A zero tap meets an Inf pixel: finite in the interior (the tap is skipped), NaN at the border.  Checked against the hand
    derivation and against the oracle, every border mode.  Zero taps keep RGBAF32 off the fused kernel."""
    rng = np.random.default_rng(51 + axis)
    img = rng.random(FLOAT_SHAPES[fmt], dtype=F32)
    if axis == 1:
        img[5, 10] = img[5, 0] = np.inf
    else:
        img[10, 5] = img[0, 5] = np.inf
    k3, one = np.array([0.5, 0.0, 0.5], F32), np.ones(1, F32)
    kx, ky = (k3, one) if axis == 1 else (one, k3)
    for border in BORDERS:
        got = zb.Image.from_numpy(img).convolve_separable(kx, ky, border_enum(zb, border)).to_numpy()
        assert _kernel(zb) == "sep_generic_f32"
        with _oracle_quiet():
            want = zo.conv_separable(img, kx, ky, border)
        assert_same_bits(got, want, (fmt, axis, border))
        line = got[5] if axis == 1 else got[:, 5]
        for i, v in _zero_tap_expected(img, axis).items():
            assert_same_bits(np.atleast_1d(line[i]), np.atleast_1d(v), (fmt, axis, border, "hand", i))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_convolve_dense_and_gaussian(zb, fmt):
    rng = np.random.default_rng(61)
    img = planted(rng, FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    for kh, kw in ((3, 3), (4, 5), (1, 7)) if fmt == "f32" else ():   # dense convolve takes F32, not Rgba(f32)
        k = (rng.standard_normal((kh, kw)) / (kh * kw)).astype(F32)
        for border in BORDERS:
            got = dev.convolve(k, border_enum(zb, border)).to_numpy()
            assert _kernel(zb) == "conv2d_generic_f32"
            with _oracle_quiet():
                assert_same_bits(got, zo.convolve(img, k, border), (fmt, kh, kw, border))
    for sigma in (0.7, 2.25):
        got = dev.gaussian_blur(sigma).to_numpy()
        with _oracle_quiet():
            want = zo.gaussian_blur(img, sigma)
        if fmt == "rgbaf32":
            assert _kernel(zb) == "fused_sep_rgbaf32"
            taps = zo.gaussian_taps(sigma)
            with _oracle_quiet():
                absconv = zo.conv_separable(np.abs(img), taps, taps, "mirror")
            assert_fma_close(got, want, absconv, taps.size, taps.size, (fmt, sigma))
        else:
            assert _kernel(zb) == "sep_generic_f32"
            assert_same_bits(got, want, (fmt, sigma))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_box_blur_and_sharpen(zb, fmt):
    img = planted(np.random.default_rng(71), FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    for radius in (1, 3):
        got = dev.box_blur(radius).to_numpy()
        assert _kernel(zb) == "sat_box_blur"
        with _oracle_quiet():
            assert_same_bits(got, zo.box_blur(img, radius), (fmt, "box", radius))
        got = dev.sharpen(radius).to_numpy()
        assert _kernel(zb) == "sat_sharpen"
        with _oracle_quiet():
            assert_same_bits(got, zo.sharpen(img, radius), (fmt, "sharpen", radius))


# ---- geometry ---------------------------------------------------------------------------------------------------------------------

SAMPLERS = [(m, 1 / 3, 1 / 3) for m in METHODS] + [("mitchell", 0.0, 0.5), ("mitchell", 1.0, 0.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_resize(zb, fmt):
    img = planted(np.random.default_rng(81), FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    for out_shape in ((29, 71), (50, 20)):
        for method, b, c in SAMPLERS:
            out = zb.Image.init(out_shape[0], out_shape[1], dev.pixfmt)
            got = dev.resize(out, method_enum(zb, method), b, c).to_numpy()
            assert _kernel(zb) == "resize_generic"
            with _oracle_quiet():
                want = zo.resize(img, out_shape, method, b, c)
            assert_same_bits(got, want, (fmt, out_shape, method, b, c))


def _cs(angle):
    a = np.float32(angle)
    return np.float32(np.cos(np.float64(a))), np.float32(np.sin(np.float64(a)))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_rotate_into(zb, fmt):
    img = planted(np.random.default_rng(91), FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    tail = FLOAT_SHAPES[fmt][2:]
    for angle in (0.4, -2.5):
        for method, b, c in SAMPLERS:
            for border in ("zero", "replicate", "mirror", "wrap"):
                out = np.full((41, 47) + tail, SENTINEL, F32)
                cs = _cs(angle)
                got = dev.rotate_into(zb.Image.from_numpy(out), np.float32(angle), method_enum(zb, method), border_enum(zb, border),
                                      cos_sin=cs, b=b, c=c).to_numpy()
                assert _kernel(zb) == "rotate_gather"
                with _oracle_quiet():
                    want = zo.rotate_into(img, out.copy(), np.float32(angle), method, border, cos_sin=cs, b=b, c=c)
                assert_same_bits(got, want, (fmt, angle, method, border))
    for angle in (np.pi / 2, np.pi, -np.pi / 2):
        for out_shape in ((60, 40), (30, 50)):
            out = np.full(out_shape + tail, SENTINEL, F32)
            got = dev.rotate_into(zb.Image.from_numpy(out), np.float32(angle)).to_numpy()
            assert _kernel(zb) == "rotate_orthogonal"
            assert_same_bits(got, zo.rotate_into(img, out.copy(), np.float32(angle)), (fmt, "orthogonal", angle, out_shape))


class _Xf:
    def __init__(self, kind, m):
        self.kind, self.m = kind, np.asarray(m, np.float32)

    def as_f32(self):
        return {"similarity": 0, "affine": 1, "projective": 2}[self.kind], self.m


WARPS = [("affine", [0.9, -0.2, 0.25, 1.1, 1.5, -2.0]), ("similarity", [0.7, 0.7, -0.7, 0.7, 3, 4]),
         ("projective", [1.0, 0.05, 2, -0.03, 0.95, 1, 1e-3, -2e-3, 1])]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_warp_extract_insert(zb, fmt):
    rng = np.random.default_rng(101)
    img = planted(rng, FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    tail = FLOAT_SHAPES[fmt][2:]
    for kind, m in WARPS:
        for method, b, c in SAMPLERS:
            out = zb.Image.init(40, 50, dev.pixfmt)
            got = dev.warp(out, _Xf(kind, m), method_enum(zb, method), b, c).to_numpy()
            assert _kernel(zb) == "warp_gather"
            with _oracle_quiet():
                want = zo.warp(img, np.zeros((40, 50) + tail, F32), kind, m, method, b, c)
            assert_same_bits(got, want, (fmt, kind, method, b, c))
    for rect, angle, out_shape in [((5.0, 4.0, 35.0, 28.0), 0.3, (20, 25)), ((-6.5, -3.0, 30.0, 50.0), -1.1, (17, 9))]:
        for method, b, c in SAMPLERS:
            for border in BORDERS:
                got = dev.extract(zb.Image.init(out_shape[0], out_shape[1], dev.pixfmt), rect, angle, method_enum(zb, method),
                                  border_enum(zb, border), b, c).to_numpy()
                assert _kernel(zb) == "extract_gather"
                with _oracle_quiet():
                    want = zo.extract(img, np.zeros(out_shape + tail, F32), rect, angle, method, border, b=b, c=c)
                assert_same_bits(got, want, (fmt, "extract", rect, method, border))
    for border in BORDERS:                                                    # copyRect: special values carried by every border
        rect = (-4.0, -3.0, 56.0, 41.0)
        got = dev.extract(zb.Image.init(44, 60, dev.pixfmt), rect, 0.0, method_enum(zb, "nearest"), border_enum(zb, border)).to_numpy()
        assert _kernel(zb) == "extract_copy_rect"
        assert_same_bits(got, zo.extract(img, np.zeros((44, 60) + tail, F32), rect, 0.0, "nearest", border), (fmt, "copy", border))
    source = planted(rng, (20, 25) + tail)
    dest = np.full((48, 60) + tail, SENTINEL, F32)
    for rect, angle in [((5.0, 4.0, 35.0, 28.0), 0.4), ((-6.5, 30.0, 30.0, 58.0), -1.2), ((3.0, 2.0, 28.0, 22.0), 0.0)]:
        for method, b, c in SAMPLERS:
            d = zb.Image.from_numpy(dest.copy())
            got = d.insert(zb.Image.from_numpy(source), rect, angle, method_enum(zb, method), b, c).to_numpy()
            assert _kernel(zb) in ("insert_gather", "insert_copy_rect")
            with _oracle_quiet():
                want = zo.insert(dest, source, rect, angle, method, b=b, c=c)
            assert_same_bits(got, want, (fmt, "insert", rect, method))


# ---- motion blur, edges, metrics ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_motion_blur(zb, fmt):
    import zignal_b200.compose as cp
    img = planted(np.random.default_rng(111), FLOAT_SHAPES[fmt])
    dev = zb.Image.from_numpy(img)
    for angle, distance in ((0.6, 7), (2.0, 4)):
        out = zb.Image.init(img.shape[0], img.shape[1], dev.pixfmt)
        got = cp.motion_blur_linear(dev, out, angle, distance).to_numpy()
        assert _kernel(zb) == "motion_line"
        with _oracle_quiet():
            assert_same_bits(got, zo.motion_blur_linear(img, angle, distance), (fmt, angle, distance))
    for spin in (False, True):
        out = zb.Image.init(img.shape[0], img.shape[1], dev.pixfmt)
        got = cp.motion_blur_radial(dev, out, 0.4, 0.6, 0.5, spin).to_numpy()
        assert _kernel(zb) == ("motion_spin" if spin else "motion_zoom")
        with _oracle_quiet():
            want = zo.motion_blur_radial(img, 0.4, 0.6, 0.5, spin)
        if not spin:
            assert_same_bits(got, want, (fmt, spin))
            continue
        # spin is not bit-exact against the oracle on finite data either (its sample positions differ in the last bits): the same
        # non-finite masks and Inf signs, and finite values within 1e-4 of the spin blur of the 3 x 3 maximum of |img|.  A bilinear
        # sample whose position moves by e changes by at most about e times the largest magnitude of its neighbourhood, and the
        # blur sums such samples; the scale is the magnitude of the terms, not of their possibly cancelling sum.
        assert np.array_equal(np.isnan(got), np.isnan(want)), (fmt, "spin NaN mask")
        assert np.array_equal(np.isposinf(got), np.isposinf(want)) and np.array_equal(np.isneginf(got), np.isneginf(want)), fmt
        a = np.pad(np.nan_to_num(np.abs(img), posinf=0.0), [(1, 1), (1, 1)] + [(0, 0)] * (img.ndim - 2), mode="edge")
        nbhd = np.max([a[i:i + img.shape[0], j:j + img.shape[1]] for i in range(3) for j in range(3)], axis=0).astype(F32)
        with _oracle_quiet():
            scale = zo.motion_blur_radial(nbhd, 0.4, 0.6, 0.5, spin).astype(np.float64)
        fin = np.isfinite(want)
        err = np.abs(got[fin].astype(np.float64) - want[fin].astype(np.float64))
        assert np.all(err <= 1e-4 * scale[fin] + 1e-6), (fmt, "spin", float(np.max(err / (scale[fin] + 1e-6))))


@pytest.mark.gpu
def test_sobel_f32(zb):
    """Sobel takes F32 (not Rgba(f32)); a NaN magnitude saturates to 255 like the oracle's clamp."""
    img = planted(np.random.default_rng(121), FLOAT_SHAPES["f32"])
    got = zb.Image.from_numpy(img).sobel().to_numpy()
    assert _kernel(zb) in ("sobel", "sobel_fused")
    with _oracle_quiet():
        assert_same_bits(got, zo.sobel(img), "f32")


def _clamped_u8(img):
    """convertColor(u8, v) of the reference for a float scalar: NaN -> 255."""
    d = np.where(np.isnan(img), 1.0, np.clip(img.astype(np.float64), 0.0, 1.0))
    return np.floor(d * 255.0 + 0.5).astype(np.uint8)


@pytest.mark.gpu
def test_canny_f32(zb):
    img = planted(np.random.default_rng(131), (70, 90))
    dev = zb.Image.from_numpy(img)
    for sigma, lo, hi in ((1.0, 20.0, 60.0), (0.0, 10.0, 40.0)):
        got = dev.canny(sigma, lo, hi).to_numpy()
        assert _kernel(zb) == "canny"
        assert_same_bits(got, zo.canny(img, sigma, lo, hi), sigma)
        assert_same_bits(got, zo.canny(_clamped_u8(img), sigma, lo, hi), ("as u8", sigma))


@pytest.mark.gpu
def test_shen_castan_f32(zb):
    img = planted(np.random.default_rng(141), (70, 90))
    dev = zb.Image.from_numpy(img)
    for o in (sco.Options(), sco.Options(use_nms=True, hysteresis=False)):
        got = dev.shen_castan(o.smooth, o.window_size, o.high_ratio, o.low_rel, o.hysteresis, o.use_nms).to_numpy()
        assert _kernel(zb) == "shen_castan"
        assert_same_bits(got, sco.shen_castan(img, o), o)
        assert_same_bits(got, sco.shen_castan(_clamped_u8(img), o), ("as u8", o))


def _same_metric(got, want, what):
    if math.isfinite(want):
        assert abs(got - want) <= 1e-12 * abs(want), (what, got, want)
    else:
        assert (math.isnan(got) and math.isnan(want)) or got == want, (what, got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_metrics(zb, fmt):
    """psnr / ssim / meanPixelError with NaN or Inf in either operand, and with only signed zeros and subnormals."""
    rng = np.random.default_rng(151)
    shape = FLOAT_SHAPES[fmt]
    clean = rng.random(shape, dtype=F32)
    other = np.clip(clean + rng.normal(0, 0.05, shape).astype(F32), 0, 1).astype(F32)
    cases = {"specials": planted(rng, shape),
             "inf_only": planted(rng, shape, np.array([np.inf, 0.25], F32), rows_full=False),
             "neg_inf_only": planted(rng, shape, np.array([-np.inf, 0.75], F32), rows_full=False),
             "zeros_subnormals": planted(rng, shape, np.array([0.0, -0.0, SUBNORMAL, -SUBNORMAL], F32))}
    for name, a in cases.items():
        for x, y, order in ((a, other, "a"), (other, a, "b")):
            dx, dy = zb.Image.from_numpy(x), zb.Image.from_numpy(y)
            with _oracle_quiet():
                want = (zo.psnr(x, y), zo.mean_pixel_error(x, y), zo.ssim(x, y))
            got_psnr = dx.psnr(dy)
            assert _kernel(zb) == "diff_sums"
            got_mpe = dx.mean_pixel_error(dy)
            got_ssim = dx.ssim(dy)
            assert _kernel(zb) == "ssim"
            for g, w, m in zip((got_psnr, got_mpe, got_ssim), want, ("psnr", "mpe", "ssim")):
                _same_metric(g, w, (fmt, name, order, m))


# ---- JPEG encode and quantize ---------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_jpeg_encode_from_float(zb, fmt):
    """Float images are encoded as Image.convert(Rgb): the bytes equal the encode of the Rgb(u8) image convert gives."""
    img = planted(np.random.default_rng(161), (45, 67) + FLOAT_SHAPES[fmt][2:])
    rgb = zo.convert(img, zo.PIX_RGB8)
    if fmt == "f32":
        assert (rgb[np.isnan(img)] == 255).all()
    dev, ref = zb.Image.from_numpy(img), zb.Image.from_numpy(rgb)
    for sub in (zb.JpegSubsampling.YUV444, zb.JpegSubsampling.YUV420):
        got = dev.encode_jpeg(90, sub)
        assert _kernel(zb).startswith("jpeg_") and _kernel(zb).endswith("_" + fmt)
        assert got == ref.encode_jpeg(90, sub), (fmt, sub)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FLOAT_SHAPES))
def test_quantize_from_float(zb, fmt):
    img = planted(np.random.default_rng(171), (45, 67) + FLOAT_SHAPES[fmt][2:])
    dev = zb.Image.from_numpy(img)
    for max_colors in (16, 256):
        got = zb.median_cut(dev, max_colors, 256)
        assert _kernel(zb) == "median_cut_histogram"
        assert np.array_equal(got, qo.median_cut(img, max_colors, 256)), max_colors
    got = zb.build_palette(dev, zb.PaletteMode.ADAPTIVE, 200)
    assert _kernel(zb) == "median_cut_histogram"
    assert np.array_equal(got, qo.build_palette(img, qo.ADAPTIVE, 200))
    pal = qo.median_cut(img, 64, 256)
    lut = zb.ColorLookupTable(pal)
    got = dev.palette_indices(lut).to_numpy()
    assert _kernel(zb) == "palette_lookup"
    assert np.array_equal(got, qo.palette_lookup(img, qo.color_lut(pal)))


# ---- host twins ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_host_twins(zb):
    rng = np.random.default_rng(181)
    img = planted(rng, (40, 48, 4))
    kx, ky = _taps(rng, 5), _taps(rng, 3)
    try:
        zb.lib().zb_set_exact_f32(1)                  # the pipelined host path runs the fused kernel
        got = zb.host_conv_separable(img, kx, ky, zb.BorderMode.REPLICATE)
    finally:
        zb.lib().zb_set_exact_f32(0)
    with _oracle_quiet():
        assert_same_bits(got, zo.conv_separable(img, kx, ky, "replicate"), "host_conv_separable")
    gray = planted(rng, (40, 48))
    k2 = (rng.standard_normal((3, 4)) / 12).astype(F32)
    with _oracle_quiet():
        assert_same_bits(zb.host_convolve(gray, k2, zb.BorderMode.WRAP), zo.convolve(gray, k2, "wrap"), "host_convolve")
        assert_same_bits(zb.host_box_blur(img, 2), zo.box_blur(img, 2), "host_box_blur")
        assert_same_bits(zb.host_sharpen(gray, 2), zo.sharpen(gray, 2), "host_sharpen")
        assert_same_bits(zb.host_gaussian_blur(gray, 1.5), zo.gaussian_blur(gray, 1.5), "host_gaussian_blur")
        assert_same_bits(zb.host_resize(img, (31, 70), zb.Interpolation.BICUBIC), zo.resize(img, (31, 70), "bicubic"), "host_resize")
    angle = np.float32(0.6)
    got = zb.host_rotate(gray, angle)
    cs = (np.float32(math.cos(float(angle))), np.float32(math.sin(float(angle))))   # the library's host libm
    with _oracle_quiet():
        want = zo.rotate(gray, angle, "bilinear", "zero", cos_sin=cs)
    assert_same_bits(got, want, "host_rotate_into")
    m = [0.9, -0.2, 0.25, 1.1, 1.5, -2.0]
    out = np.zeros((35, 45, 4), F32)
    with _oracle_quiet():
        assert_same_bits(zb.host_warp(img, out, _Xf("affine", m)), zo.warp(img, np.zeros_like(out), "affine", m, "bilinear"), "host_warp")


# ---- 8-bit-only entry points refuse float images ----------------------------------------------------------------------------------

@pytest.mark.gpu
def test_eight_bit_entry_points_refuse_f32(zb):
    L = zb.lib()
    img = zb.Image.from_numpy(np.random.default_rng(191).random((16, 20), dtype=F32))
    out = zb.Image.init(16, 20, zb.PixFmt.F32)
    a, d = img._zb(), out._zb()
    UNSUPPORTED = 3
    F = int(zb.PixFmt.F32)
    counts = (C.c_uint32 * 1024)()
    sums = (C.c_uint64 * 11)()
    pal = (C.c_uint8 * 768)()
    lut = (C.c_uint8 * 32768)()
    fdm = C.c_void_p()
    from zignal_b200.image import _np_image
    h_src, h_tgt = np.zeros((8, 8), F32), np.zeros((8, 8), F32)
    calls = {
        "zb_order_blur": lambda: L.zb_order_blur(a, d, F, 1, 0, C.c_double(0.5), 2, None),
        "zb_histogram": lambda: L.zb_histogram(a, F, counts, None),
        "zb_autocontrast": lambda: L.zb_autocontrast(d, F, C.c_float(0.0), None),
        "zb_equalize": lambda: L.zb_equalize(d, F, None),
        "zb_dither": lambda: L.zb_dither(d, F, pal, 16, lut, 1, None),
        "zb_fdm_create": lambda: L.zb_fdm_create(C.byref(fdm), F),
        "zb_fdm_moments": lambda: L.zb_fdm_moments(a, F, 0, sums, None),
        "zb_host_fdm_match": lambda: L.zb_host_fdm_match(_np_image(h_src), _np_image(h_tgt), F),
    }
    assert set(calls) == {n for n, cls in FLOAT_ENTRY_POINTS.items() if cls == "8-bit only"}
    for name, call in calls.items():
        assert call() == UNSUPPORTED, name
    assert not fdm.value

