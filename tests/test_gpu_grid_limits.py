"""Tall images and long matrices past the 65,535 limit of gridDim.y.

A kernel that tiles rows needs one grid row per tile.  Launched with the tile index straight in gridDim.y it is refused once an image
has more than 65,535 tiles: 524,281 rows at 8 rows per tile, 2,097,121 at 32, 4,194,241 at 64.  Every entry point below runs at the
last height that fits such a grid and the first that does not, on the kernel named by zb_last_kernel(), against the oracle and at
the bar of that family's own test (bit-exact for integer formats and the bit-exact f32 paths; 1e-12 relative for SSIM; 2e-6 / 1e-12
of max|C| for GEMM).  Images stay 1-16 columns wide (at most ~70 MB) so the oracle stays cheap.  The kernels that spread one grid row
per image row over (y, z) are checked at the seams of that split (65,535 / 65,536 / 131,071 / 196,606 rows).

Cost: the whole file (77 tests, oracle included) ran in 78 s on one H100 80GB HBM3 at a 700 W power limit.
"""
import numpy as np
import pytest

import binary_oracle as bo
import oracle_lib as zo
import shen_castan_oracle as sco
from gpu_utils import rand_image

pytestmark = pytest.mark.gpu

H8 = [524_280, 524_281]          # 8 rows per tile: 65,535 tiles, then 65,536
H32 = [2_097_120, 2_097_121]     # 32 rows per tile
H64 = [4_194_240, 4_194_241]     # 64 rows per tile
SEAMS = [65_535, 65_536, 131_071, 196_606]   # row_grid: one z-slice, two slices, the first row of a third, two full slices
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    yield zb
    zb.lib().zb_set_force_generic(0)
    zb.lib().zb_tune(b"sobel.tile", 1)


def _kernel(zb):
    return zb.lib().zb_last_kernel().decode()


def _img(rows, cols, fmt, seed):
    rng = np.random.default_rng(seed)
    tail = {"u8": (), "f32": (), "rgb8": (3,), "rgba8": (4,)}[fmt]
    return rand_image(rng, (rows, cols) + tail, np.float32 if fmt == "f32" else np.uint8)


class _Xf:
    def __init__(self, kind, m):
        self.kind, self.m = kind, np.asarray(m, np.float32)

    def as_f32(self):
        return {"similarity": 0, "affine": 1, "projective": 2}[self.kind], self.m


def _in_view(zb, img, fill, pad=(3, 2)):
    """`img` as a strided device view inside a bigger buffer of `fill` (rows / cols offset by pad, ragged stride)."""
    t, l = pad
    base = np.full((img.shape[0] + t + 2, img.shape[1] + l + 3) + img.shape[2:], fill, img.dtype)
    base[t:t + img.shape[0], l:l + img.shape[1]] = img
    dev = zb.Image.from_numpy(base)
    return dev, dev.view(zb.Rectangle(l, t, l + img.shape[1], t + img.shape[0]))


def _check_view_case(zb, img, run, want):
    """run(src_view, dst_view) from a strided source view into a strided destination view whose buffer holds SENTINEL around it:
    the view must equal `want` and nothing outside it may change (the widened grid neither skips nor overruns rows)."""
    _, sv = _in_view(zb, img, 0x5A if img.dtype == np.uint8 else -3.0)
    proto = np.zeros(want.shape, want.dtype)
    fill = SENTINEL if want.dtype == np.uint8 else np.float32(-7.5)
    dbase, dv = _in_view(zb, proto, fill, pad=(2, 1))
    run(sv, dv)
    got = dbase.to_numpy()
    t, l = 2, 1
    assert np.array_equal(got[t:t + want.shape[0], l:l + want.shape[1]], want)
    outside = np.ones(got.shape[:2], bool)
    outside[t:t + want.shape[0], l:l + want.shape[1]] = False
    assert (got[outside] == fill).all()


# ---- 8 rows per tile ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rows", H8)
def test_convolve_generic_f32(zb, rows):
    img = _img(rows, 5, "f32", rows)
    k = np.random.default_rng(1).standard_normal((3, 3)).astype(np.float32) / 9
    got = zb.Image.from_numpy(img).convolve(k, zb.BorderMode.MIRROR).to_numpy()
    assert _kernel(zb) == "conv2d_generic_f32"
    assert np.array_equal(got, zo.convolve(img, k, "mirror"))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "rgb8"])
def test_convolve_generic_u8_9x9(zb, rows, fmt):
    img = _img(rows, 6, fmt, rows + 1)
    k = np.random.default_rng(2).standard_normal((9, 9)).astype(np.float32) / 40
    got = zb.Image.from_numpy(img).convolve(k, zb.BorderMode.REPLICATE).to_numpy()
    assert _kernel(zb) == "conv2d_generic_u8"
    assert np.array_equal(got, zo.convolve(img, k, "replicate"))


def test_convolve_generic_strided_views(zb):
    rows = H8[1]
    k = np.random.default_rng(3).standard_normal((3, 3)).astype(np.float32) / 9
    for fmt in ("f32", "u8"):
        img = _img(rows, 7, fmt, 4)
        kk = k if fmt == "f32" else np.random.default_rng(5).standard_normal((9, 9)).astype(np.float32) / 40

        def run(sv, dv):
            sv.convolve(kk, zb.BorderMode.WRAP, out=dv)
            assert _kernel(zb) == ("conv2d_generic_f32" if fmt == "f32" else "conv2d_generic_u8")
        _check_view_case(zb, img, run, zo.convolve(img, kk, "wrap"))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_canny(zb, rows, fmt):
    img = _img(rows, 8, fmt, rows + 2)
    got = zb.Image.from_numpy(img).canny(1.0, 20.0, 60.0).to_numpy()
    assert _kernel(zb) == "canny"
    assert np.array_equal(got, zo.canny(img, 1.0, 20.0, 60.0))


@pytest.mark.parametrize("rows", H8)
def test_sobel_fused(zb, rows):
    img = (_img(rows, 9, "f32", rows + 3) * 255.0).astype(np.float32)
    got = zb.Image.from_numpy(img).sobel().to_numpy()
    assert _kernel(zb) == "sobel_fused"
    assert np.array_equal(got, zo.sobel(img))
    u8 = _img(rows, 9, "rgb8", rows + 4)
    zb.lib().zb_tune(b"sobel.tile", 0)
    try:
        got = zb.Image.from_numpy(u8).sobel().to_numpy()
        assert _kernel(zb) == "sobel_fused"
    finally:
        zb.lib().zb_tune(b"sobel.tile", 1)
    assert np.array_equal(got, zo.sobel(u8))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_shen_castan(zb, rows, fmt):
    img = _img(rows, 8, fmt, rows + 5)
    o = sco.Options()
    got = zb.Image.from_numpy(img).shen_castan(o.smooth, o.window_size, o.high_ratio, o.low_rel, o.hysteresis, o.use_nms).to_numpy()
    assert _kernel(zb) == "shen_castan"
    assert np.array_equal(got, sco.shen_castan(img, o))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["rgb8", "u8"])
def test_order_blur(zb, rows, fmt):
    img = _img(rows, 5, fmt, rows + 6)
    got = zb.Image.from_numpy(img).median_blur(1).to_numpy()
    assert _kernel(zb) == "order_statistic"
    assert np.array_equal(got, zo.order_blur(img, 1, "percentile", 0.5, "mirror"))
    got = zb.Image.from_numpy(img).midpoint_blur(2, zb.BorderMode.WRAP).to_numpy()
    assert np.array_equal(got, zo.order_blur(img, 2, "midpoint", 0.0, "wrap"))


def test_order_blur_strided_views(zb):
    img = _img(H8[1], 6, "rgb8", 7)

    def run(sv, dv):
        sv.median_blur(1, out=dv)
        assert _kernel(zb) == "order_statistic"
    _check_view_case(zb, img, run, zo.order_blur(img, 1, "percentile", 0.5, "mirror"))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_motion_blur(zb, rows, fmt):
    from zignal_b200.compose import motion_blur_linear, motion_blur_radial
    img = _img(rows, 4, fmt, rows + 8)
    dev = zb.Image.from_numpy(img)
    got = motion_blur_linear(dev, zb.Image.init_like(dev), 0.7, 5).to_numpy()
    assert _kernel(zb) == "motion_line"
    assert np.array_equal(got, zo.motion_blur_linear(img, 0.7, 5))
    got = motion_blur_radial(dev, zb.Image.init_like(dev), 0.5, 0.999, 0.3).to_numpy()
    assert _kernel(zb) == "motion_zoom"
    assert np.array_equal(got, zo.motion_blur_radial(img, 0.5, 0.999, 0.3))


def test_motion_blur_strided_views(zb):
    from zignal_b200.compose import motion_blur_linear
    img = _img(H8[1], 5, "u8", 9)

    def run(sv, dv):
        motion_blur_linear(sv, dv, -1.1, 7)
        assert _kernel(zb) == "motion_line"
    _check_view_case(zb, img, run, zo.motion_blur_linear(img, -1.1, 7))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_rotate_orthogonal_into_tall_destination(zb, rows, fmt):
    """A wide image turned by 90 / 270 degrees: the destination is the tall one."""
    img = _img(5, rows, fmt, rows + 10)
    dev = zb.Image.from_numpy(img)
    for angle in (np.pi / 2, 3 * np.pi / 2):
        got = dev.rotate(np.float32(angle)).to_numpy()
        assert _kernel(zb) == "rotate_orthogonal"
        assert got.shape[:2] == (rows, 5)
        assert np.array_equal(got, zo.rotate(img, np.float32(angle)))


@pytest.mark.parametrize("rows", H8)
def test_rotate_orthogonal_tall_source(zb, rows):
    img = _img(rows, 3, "rgb8", rows + 11)
    got = zb.Image.from_numpy(img).rotate(np.float32(np.pi)).to_numpy()
    assert _kernel(zb) == "rotate_orthogonal"
    assert np.array_equal(got, zo.rotate(img, np.float32(np.pi)))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_warp(zb, rows, fmt):
    img = _img(rows, 6, fmt, rows + 12)
    dev = zb.Image.from_numpy(img)
    m = [0.9, -0.2, 0.25, 1.1, 1.5, -2.0]
    out = zb.Image.init(rows, 4, dev.pixfmt)
    got = dev.warp(out, _Xf("affine", m), zb.Interpolation.BILINEAR).to_numpy()
    assert _kernel(zb) == "warp_gather"
    assert np.array_equal(got, zo.warp(img, np.zeros((rows, 4) + img.shape[2:], img.dtype), "affine", m, "bilinear"))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_extract(zb, rows, fmt):
    img = _img(rows, 6, fmt, rows + 13)
    dev = zb.Image.from_numpy(img)
    rect, angle = (0.5, 1.0, 5.5, rows - 2.0), 0.001
    out = zb.Image.init(rows, 5, dev.pixfmt)
    got = dev.extract(out, rect, angle, zb.Interpolation.BILINEAR, zb.BorderMode.MIRROR).to_numpy()
    assert _kernel(zb) == "extract_gather"
    assert np.array_equal(got, zo.extract(img, np.zeros((rows, 5) + img.shape[2:], img.dtype), rect, angle, "bilinear", "mirror"))


@pytest.mark.parametrize("rows", H8)
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_insert(zb, rows, fmt):
    dest = _img(rows, 6, fmt, rows + 14)
    source = _img(rows // 3, 4, fmt, rows + 15)
    rect, angle = (0.5, -1.0, 5.5, rows + 1.0), 0.0005
    dev = zb.Image.from_numpy(dest)
    got = dev.insert(zb.Image.from_numpy(source), rect, angle, zb.Interpolation.BILINEAR).to_numpy()
    assert _kernel(zb) == "insert_gather"
    assert np.array_equal(got, zo.insert(dest, source, rect, angle, "bilinear"))


def test_insert_strided_views(zb):
    rows = H8[1]
    dest = _img(rows, 6, "u8", 16)
    source = _img(rows // 3, 4, "u8", 17)
    rect, angle = (0.5, -1.0, 5.5, rows + 1.0), 0.0005
    want = zo.insert(dest, source, rect, angle, "bilinear")
    dbase, dv = _in_view(zb, dest, SENTINEL)
    _, sv = _in_view(zb, source, 0x5A)
    dv.insert(sv, rect, angle, zb.Interpolation.BILINEAR)
    assert _kernel(zb) == "insert_gather"
    got = dbase.to_numpy()
    assert np.array_equal(got[3:3 + rows, 2:8], want)
    outside = np.ones(got.shape, bool)
    outside[3:3 + rows, 2:8] = False
    assert (got[outside] == SENTINEL).all()


@pytest.mark.parametrize("rows", H8)
def test_insert_from_another_pixel_type(zb, rows):
    """An 8-bit gray source inserted into an f32 image (the mixed kernel): the oracle inserts into a 0 and a 255 canvas to find the
    pixels the rectangle writes, and converts those."""
    dest = _img(rows, 6, "f32", rows + 18)
    source = _img(rows // 3, 4, "u8", rows + 19)
    rect, angle = (0.5, -1.0, 5.5, rows + 1.0), 0.0005
    d = zb.Image.from_numpy(dest)
    d.insert(zb.Image.from_numpy(source), rect, angle, zb.Interpolation.BILINEAR)
    assert _kernel(zb) == "insert_mixed"
    s0 = zo.insert(np.zeros(dest.shape, np.uint8), source, rect, angle, "bilinear")
    s1 = zo.insert(np.full(dest.shape, 255, np.uint8), source, rect, angle, "bilinear")
    written = s0 == s1
    want = dest.copy()
    want[written] = zo.convert(s0, zo.PIX_F32)[written]
    assert np.array_equal(d.to_numpy(), want)


@pytest.mark.parametrize("rows", [h + 10 for h in H8])   # SSIM tiles the rows - 10 window origins
@pytest.mark.parametrize("fmt", ["u8", "f32"])
def test_ssim(zb, rows, fmt):
    rng = np.random.default_rng(rows + 20)
    a = _img(rows, 12, fmt, rows + 21)
    if fmt == "u8":
        b = np.clip(a.astype(np.int32) + rng.integers(-25, 26, a.shape), 0, 255).astype(np.uint8)
    else:
        b = np.clip(a + rng.normal(0, 0.05, a.shape).astype(np.float32), 0, 1).astype(np.float32)
    da, db = zb.Image.from_numpy(a), zb.Image.from_numpy(b)
    got = da.ssim(db)
    assert _kernel(zb) == "ssim"
    want = zo.ssim(a, b)
    assert abs(got - want) <= 1e-12 * abs(want), (got, want)
    assert da.ssim(db) == got   # fixed block order, host-side final sum


# ---- 32 rows per tile -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rows", H32)
def test_morphology(zb, rows):
    img = _img(rows, 7, "u8", rows + 22)
    img[img < 140] = 0
    cross = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], np.uint8)
    dev = zb.Image.from_numpy(img)
    got = dev.dilate_binary(cross, 1).to_numpy()
    assert _kernel(zb) == "morph_binary"
    assert np.array_equal(got, bo.morph_binary(img, cross, 1, "dilate"))
    got = dev.close_binary(np.ones((5, 3), np.uint8), 2).to_numpy()
    assert np.array_equal(got, bo.morph_binary(img, np.ones((5, 3), np.uint8), 2, "close"))


@pytest.mark.parametrize("rows", H32)
def test_sobel_tile_u8(zb, rows):
    img = _img(rows, 4, "u8", rows + 23)
    got = zb.Image.from_numpy(img).sobel().to_numpy()
    assert _kernel(zb) == "sobel_tile_u8"
    assert np.array_equal(got, zo.sobel(img))


@pytest.mark.parametrize("rows", H32)
def test_convolve_tile_u8(zb, rows):
    img = _img(rows, 4, "u8", rows + 24)
    k = np.random.default_rng(6).standard_normal((3, 3)).astype(np.float32) / 9
    got = zb.Image.from_numpy(img).convolve(k, zb.BorderMode.MIRROR).to_numpy()
    assert _kernel(zb) == "conv2d_tile_u8"
    assert np.array_equal(got, zo.convolve(img, k, "mirror"))


# ---- 64 rows per tile -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("rows", H64)
def test_box_fused(zb, rows):
    img = _img(rows, 4, "u8", rows + 25)
    dev = zb.Image.from_numpy(img)
    got = dev.box_blur(2).to_numpy()
    assert _kernel(zb) == "box_fused_blur"
    assert np.array_equal(got, zo.box_blur(img, 2))
    got = dev.sharpen(3).to_numpy()
    assert _kernel(zb) == "box_fused_sharpen"
    assert np.array_equal(got, zo.sharpen(img, 3))
    got = dev.threshold_adaptive_mean(2, 1.5).to_numpy()
    assert _kernel(zb) == "box_fused_threshold"
    assert np.array_equal(got, bo.threshold_adaptive_mean(img, 2, 1.5))


@pytest.mark.parametrize("rows", H64)
def test_convolve_separable_tile_u8(zb, rows):
    img = _img(rows, 4, "u8", rows + 26)
    kx = np.array([-0.1, 0.3, 0.6, 0.3, -0.1], np.float32)       # a negative tap: the 64-row tile, not the dot-product variant
    ky = np.array([0.2, 0.6, 0.2], np.float32)
    got = zb.Image.from_numpy(img).convolve_separable(kx, ky, zb.BorderMode.MIRROR).to_numpy()
    assert _kernel(zb) == "sep_tile_u8"
    assert np.array_equal(got, zo.conv_separable(img, kx, ky, "mirror"))


@pytest.mark.parametrize("rows", H64)
@pytest.mark.parametrize("fmt", ["rgba8", "f32"])
def test_rotate_gather_into_tall_destination(zb, rows, fmt):
    """A non-orthogonal angle into a tall, narrow destination: 64 destination rows per block (8 row groups x 8 rows per thread)."""
    img = _img(9, 4, fmt, rows + 27)
    fill = _img(rows, 4, fmt, rows + 28)
    out = zb.Image.from_numpy(fill)
    zb.Image.from_numpy(img).rotate_into(out, np.float32(0.3))
    assert _kernel(zb) == "rotate_gather"      # (Rgba8: the tile kernel takes destinations up to 16,384 rows only)
    assert np.array_equal(out.to_numpy(), zo.rotate_into(img, fill.copy(), np.float32(0.3)))


def test_rotate_tile_rgba8_tallest_destination(zb):
    img = _img(40, 16, "rgba8", 29)
    fill = _img(16_384, 4, "rgba8", 30)
    out = zb.Image.from_numpy(fill)
    zb.Image.from_numpy(img).rotate_into(out, np.float32(1.1))
    assert _kernel(zb) == "rotate_tile_rgba8"
    assert np.array_equal(out.to_numpy(), zo.rotate_into(img, fill.copy(), np.float32(1.1)))


# ---- one grid row per image row: the (y, z) seams of row_grid -------------------------------------------------------------------

@pytest.mark.parametrize("rows", SEAMS)
def test_row_grid_seams(zb, rows):
    L = zb.lib()
    g = _img(rows, 5, "u8", rows + 31)
    rgb = _img(rows, 3, "rgb8", rows + 32)
    f = _img(rows, 5, "f32", rows + 33)
    dg, drgb, df = zb.Image.from_numpy(g), zb.Image.from_numpy(rgb), zb.Image.from_numpy(f)
    assert np.array_equal(drgb.convert(zb.PixFmt.U8).to_numpy(), zo.convert(rgb, zo.PIX_U8))
    assert _kernel(zb) == "convert"
    assert np.array_equal(dg.convert(zb.PixFmt.F32).to_numpy(), zo.convert(g, zo.PIX_F32))
    # both resizers: the 8-bit plane kernel and the generic one
    for src, dev in ((rgb, drgb), (f, df)):
        out = zb.Image.init(rows + 7, 4, dev.pixfmt)
        got = dev.resize(out, zb.Interpolation.BILINEAR).to_numpy()
        assert _kernel(zb) == ("resize_plane_u8" if src.dtype == np.uint8 else "resize_generic")
        assert np.array_equal(got, zo.resize(src, (rows + 7, 4), "bilinear"))
    # the two-pass separable convolution
    kx, ky = np.array([0.25, 0.5, 0.25], np.float32), np.array([0.1, 0.2, 0.4, 0.2, 0.1], np.float32)
    L.zb_set_force_generic(1)
    try:
        for src, dev in ((g, dg), (f, df)):
            got = dev.convolve_separable(kx, ky, zb.BorderMode.MIRROR).to_numpy()
            assert _kernel(zb) == ("sep_generic_u8" if src.dtype == np.uint8 else "sep_generic_f32")
            assert np.array_equal(got, zo.conv_separable(src, kx, ky, "mirror"))
        got = dg.sobel().to_numpy()          # gray pass, generic convolutions, magnitude pass
        assert _kernel(zb) == "sobel"
        assert np.array_equal(got, zo.sobel(g))
    finally:
        L.zb_set_force_generic(0)
    # sat_eval: box blur of a float image
    got = df.box_blur(2).to_numpy()
    assert _kernel(zb) == "sat_box_blur"
    assert np.array_equal(got, zo.box_blur(f, 2))
    # Canny's gray and finalize passes
    got = drgb.canny(0.0, 30.0, 90.0).to_numpy()
    assert _kernel(zb) == "canny"
    assert np.array_equal(got, zo.canny(rgb, 0.0, 30.0, 90.0))


# ---- GEMM: 64 rows of M per block -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("m", [4_194_241, 4_194_304])
@pytest.mark.parametrize("dtype,tol", [(np.float32, 2e-6), (np.float64, 1e-12)])
def test_gemm_long_m(zb, m, dtype, tol):
    from zignal_b200.matrix import gemm
    rng = np.random.default_rng(m)
    k = 3
    for n in (2, 3):
        for ta in (False, True):
            for tb in (False, True):
                a = rng.standard_normal((k, m) if ta else (m, k)).astype(dtype)
                b = rng.standard_normal((n, k) if tb else (k, n)).astype(dtype)
                c = rng.standard_normal((m, n)).astype(dtype)
                a64, b64 = (a.T if ta else a).astype(np.float64), (b.T if tb else b).astype(np.float64)
                got = gemm(a, b, ta, tb, 0.5, 2.0, c)
                assert _kernel(zb) == ("gemm_f32_acc64" if dtype == np.float32 else "gemm_f64")
                ref = 0.5 * (a64 @ b64) + 2.0 * c.astype(np.float64)
                assert np.abs(got - ref).max() / np.abs(ref).max() <= tol, (n, ta, tb)
                got0 = gemm(a, b, ta, tb, 1.0, 0.0, None)
                ref0 = a64 @ b64
                assert np.abs(got0 - ref0).max() / np.abs(ref0).max() <= tol, (n, ta, tb)


@pytest.mark.parametrize("dtype,tol", [(np.float32, 2e-6), (np.float64, 1e-12)])
def test_pca_transform_of_a_2048_squared_image(zb, dtype, tol):
    """Pca.transform of the 4,194,304 RGB pixels of one 2048 x 2048 image (M = 4,194,304, K = 3)."""
    from zignal_b200.pca import Pca
    rng = np.random.default_rng(4)
    x = (rng.random((2048 * 2048, 3)) * 255.0).astype(dtype)
    x[:, 1] = (0.6 * x[:, 0] + 0.4 * x[:, 1]).astype(dtype)
    p = Pca(dtype)
    p.fit(x[:50_000])
    got = p.transform(x)
    assert got.shape == (x.shape[0], p.num_components)
    want = zo.pca_transform(x, p.mean, p.components)
    assert np.abs(got - want).max() / np.abs(want).max() <= tol
