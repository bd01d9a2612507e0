"""Parity of the CUDA convolution paths (generic two-pass, fused TMA kernel, dense 2-D) against the
oracle, through the C ABI.  Integer formats: bit-exact.  f32: bit-exact for the generic path and the
fused kernel's exact mode, <= 1e-5 relative (north_star tolerance) for the fused FFMA mode."""
import numpy as np
import pytest

import oracle_lib as zo
from gpu_utils import BORDERS, border_enum, golden, rand_image, rel_err, sha

pytestmark = pytest.mark.gpu
TOL_F32 = 1e-5  # BASELINE.json north_star: "within 1e-5 relative for f32 paths"


@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    yield zb
    zb.lib().zb_set_exact_f32(0)
    zb.lib().zb_set_force_generic(0)


def _dp_eligible(kx, ky):
    """The dp4a / dp2a variant of the Rgba8 kernel takes kernels whose Q8 taps are bytes and whose horizontal sums fit 16 bits."""
    qx = np.round(np.asarray(kx, np.float32) * np.float32(256)).astype(np.int64)
    qy = np.round(np.asarray(ky, np.float32) * np.float32(256)).astype(np.int64)
    return bool(qx.min() >= 0 and qx.max() <= 255 and qy.min() >= 0 and qy.max() <= 255 and int(qx.sum()) * 255 <= 65535)


def _taps(rng, n):
    k = (rng.random(n) + 0.05).astype(np.float32)
    return (k / k.sum()).astype(np.float32)


FORMATS = [((37, 53), np.uint8), ((31, 47, 3), np.uint8), ((40, 41, 4), np.uint8), ((37, 53), np.float32), ((33, 29, 4), np.float32)]


@pytest.mark.parametrize("shape,dtype", FORMATS)
@pytest.mark.parametrize("border", BORDERS)
def test_generic_separable_bit_exact(zb, shape, dtype, border):
    rng = np.random.default_rng(abs(hash((shape, str(dtype), border))) % 2**32)
    zb.lib().zb_set_force_generic(1)
    try:
        for nx, ny in [(1, 1), (3, 5), (7, 7), (4, 6), (15, 15), (31, 3)]:
            img = rand_image(rng, shape, dtype)
            kx, ky = _taps(rng, nx), _taps(rng, ny)
            got = zb.Image.from_numpy(img).convolve_separable(kx, ky, border_enum(zb, border)).to_numpy()
            assert np.array_equal(got, zo.conv_separable(img, kx, ky, border)), (nx, ny)
    finally:
        zb.lib().zb_set_force_generic(0)


def test_generic_separable_extreme_taps_use_wide_accumulators(zb):
    rng = np.random.default_rng(5)
    img = rand_image(rng, (20, 23), np.uint8)
    for scale in (1.0, 300.0, 40000.0):  # i32 / mixed / i64 accumulator paths, saturated i32 temp
        kx = (rng.standard_normal(5) * scale).astype(np.float32)
        ky = (rng.standard_normal(5) * scale).astype(np.float32)
        got = zb.Image.from_numpy(img).convolve_separable(kx, ky, zb.BorderMode.MIRROR).to_numpy()
        assert np.array_equal(got, zo.conv_separable(img, kx, ky, "mirror")), scale


def test_negligible_taps_follow_interior_only_skip_rule(zb):
    # convolution.zig:459-467: |k| < 1e-10 skipped in the interior only; finite data -> identical either way
    rng = np.random.default_rng(6)
    img = rand_image(rng, (30, 40, 4), np.float32)
    k = np.array([0.25, 1e-12, 0.5, 0.0, 0.25], np.float32)
    got = zb.Image.from_numpy(img).convolve_separable(k, k, zb.BorderMode.MIRROR).to_numpy()
    assert zb.lib().zb_last_kernel().decode().startswith("sep_generic")
    assert np.array_equal(got, zo.conv_separable(img, k, k, "mirror"))


@pytest.mark.parametrize("rows,cols", [(64, 64), (96, 520), (300, 777), (513, 1030), (40, 16), (257, 263)])
@pytest.mark.parametrize("border", BORDERS)
def test_fused_rgbaf32_exact_and_fma(zb, rows, cols, border):
    rng = np.random.default_rng(rows * 131 + cols)
    L = zb.lib()
    for half in (1, 2, 4, 7, 8):
        img = rand_image(rng, (rows, cols, 4), np.float32)
        k = _taps(rng, 2 * half + 1)
        want = zo.conv_separable(img, k, k, border)
        dev = zb.Image.from_numpy(img)
        L.zb_set_exact_f32(1)
        got = dev.convolve_separable(k, k, border_enum(zb, border)).to_numpy()
        assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32_exact"
        assert np.array_equal(got, want), ("exact", half)
        L.zb_set_exact_f32(0)
        got = dev.convolve_separable(k, k, border_enum(zb, border)).to_numpy()
        assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32"
        assert rel_err(got, want) <= TOL_F32, ("fma", half)


@pytest.mark.parametrize("rows,cols", [(64, 256), (96, 520), (300, 776), (40, 16), (72, 264), (513, 1032)])
def test_fused_rgbaf32_x_border_copies(zb, rows, cols):
    """.replicate / .mirror with cols % 8 == 0: the 8 columns either side of the image are produced by 16-byte copies inside the
    TMA stage (host-resolved source columns) instead of the generic patch pass.  Both ways must give the same bits (15, 17 and 7
    taps; fma and exact arithmetic) and match the oracle."""
    L = zb.lib()
    rng = np.random.default_rng(rows + cols)
    img = rand_image(rng, (rows, cols, 4), np.float32)
    dev = zb.Image.from_numpy(img)
    try:
        for border in ("mirror", "replicate"):
            for half in (7, 8, 3):
                k = _taps(rng, 2 * half + 1)
                for exact in (0, 1):
                    L.zb_set_exact_f32(exact)
                    res = []
                    for knob in (1, 0):
                        L.zb_tune(b"conv.edge_fast", knob)
                        res.append(dev.convolve_separable(k, k, border_enum(zb, border)).to_numpy())
                        assert L.zb_last_kernel().decode().startswith("fused_sep_rgbaf32")
                    assert np.array_equal(res[0], res[1]), (border, half, exact)
                    want = zo.conv_separable(img, k, k, border)
                    assert (np.array_equal(res[0], want) if exact else rel_err(res[0], want) <= TOL_F32), (border, half, exact)
    finally:
        L.zb_set_exact_f32(0)
        L.zb_tune(b"conv.edge_fast", 1)


@pytest.mark.parametrize("rows,cols", [(64, 64), (96, 520), (300, 776), (513, 1032), (40, 16), (257, 260)])
@pytest.mark.parametrize("border", BORDERS)
def test_fused_rgba8_bit_exact(zb, rows, cols, border):
    rng = np.random.default_rng(rows * 7 + cols)
    L = zb.lib()
    for half in (1, 2, 4, 7, 8):
        img = rand_image(rng, (rows, cols, 4), np.uint8)
        for k in (_taps(rng, 2 * half + 1), (rng.standard_normal(2 * half + 1) * 0.4).astype(np.float32)):  # positive and signed taps
            want = zo.conv_separable(img, k, k, border)
            # three pipelines, one result: dp4a / dp2a (byte taps only), exact integers on FFMA (when provably exact), IMAD
            for dp, fmath in ((1, 1), (0, 1), (0, 0)):
                L.zb_tune(b"conv.u8_dp", dp)
                L.zb_tune(b"conv.u8_fmath", fmath)
                got = zb.Image.from_numpy(img).convolve_separable(k, k, border_enum(zb, border)).to_numpy()
                name = L.zb_last_kernel().decode()
                assert name.startswith("fused_sep_rgba8"), name
                assert (name == "fused_sep_rgba8_dp") == bool(dp and _dp_eligible(k, k)), (name, dp)
                assert np.array_equal(got, want), (half, dp, fmath, name)
    L.zb_tune(b"conv.u8_fmath", 1)
    L.zb_tune(b"conv.u8_dp", 1)


def test_fused_rgba8_views_fallbacks_and_gaussian(zb):
    rng = np.random.default_rng(77)
    L = zb.lib()
    img = rand_image(rng, (200, 304, 4), np.uint8)
    big = zb.Image.from_numpy(img)
    v = big.view(zb.Rectangle(8, 5, 292, 190))          # offset 8 px = 32 B: still 16-byte aligned, pitch 304 px
    crop = np.ascontiguousarray(img[5:190, 8:292])
    out_big = zb.Image.from_numpy(np.full((220, 312, 4), 9, np.uint8))
    ov = out_big.view(zb.Rectangle(3, 2, 287, 187))
    kx, ky = _taps(rng, 6), _taps(rng, 15)
    v.convolve_separable(kx, ky, zb.BorderMode.MIRROR, out=ov)
    assert L.zb_last_kernel().decode() == ("fused_sep_rgba8_dp" if _dp_eligible(kx, ky) else "fused_sep_rgba8_f")
    full = out_big.to_numpy()
    assert np.array_equal(full[2:187, 3:287], zo.conv_separable(crop, kx, ky, "mirror"))
    mask = np.ones(full.shape[:2], bool)
    mask[2:187, 3:287] = False
    assert np.all(full[mask] == 9)
    # a view that breaks TMA alignment (offset 3 px) takes the shared-memory tile kernel; taps that need i64 accumulators the two-pass path
    v2 = big.view(zb.Rectangle(3, 0, 299, 100))
    got = v2.convolve_separable(kx, ky, zb.BorderMode.WRAP).to_numpy()
    assert L.zb_last_kernel().decode() in ("sep_tile_u8", "sep_tile_u8_dp")
    assert np.array_equal(got, zo.conv_separable(np.ascontiguousarray(img[0:100, 3:299]), kx, ky, "wrap"))
    huge = (rng.standard_normal(5) * 3000).astype(np.float32)
    got = big.convolve_separable(huge, huge, zb.BorderMode.MIRROR).to_numpy()
    assert L.zb_last_kernel().decode() == "sep_generic_u8"
    assert np.array_equal(got, zo.conv_separable(img, huge, huge, "mirror"))
    for sigma in (0.5, 1.0, 2.25):
        got = big.gaussian_blur(sigma).to_numpy()
        g = zb.gaussian_taps(sigma)
        assert L.zb_last_kernel().decode() == ("fused_sep_rgba8_dp" if _dp_eligible(g, g) else "fused_sep_rgba8_f")
        assert np.array_equal(got, zo.gaussian_blur(img, sigma)), sigma


def test_fused_handles_views_even_and_unequal_kernels(zb):
    rng = np.random.default_rng(7)
    L = zb.lib()
    img = rand_image(rng, (200, 300, 4), np.float32)
    big = zb.Image.from_numpy(img)
    v = big.view(zb.Rectangle(8, 5, 290, 190))
    crop = np.ascontiguousarray(img[5:190, 8:290])
    out_big = zb.Image.from_numpy(np.full((220, 310, 4), 7.0, np.float32))
    out_v = out_big.view(zb.Rectangle(3, 2, 285, 187))
    for kx, ky in [(_taps(rng, 6), _taps(rng, 5)), (_taps(rng, 3), _taps(rng, 15)), (_taps(rng, 16), _taps(rng, 2))]:
        L.zb_set_exact_f32(1)
        v.convolve_separable(kx, ky, zb.BorderMode.MIRROR, out=out_v)
        assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32_exact"
        got_full = out_big.to_numpy()
        assert np.array_equal(got_full[2:187, 3:285], zo.conv_separable(crop, kx, ky, "mirror"))
        mask = np.ones(got_full.shape[:2], bool)
        mask[2:187, 3:285] = False
        assert np.all(got_full[mask] == 7.0), "pixels outside the destination view were touched"
    L.zb_set_exact_f32(0)


def test_in_place_separable(zb):
    rng = np.random.default_rng(8)
    for shape, dtype in [((64, 70, 4), np.float32), ((50, 61, 4), np.uint8)]:
        img = rand_image(rng, shape, dtype)
        k = _taps(rng, 7)
        dev = zb.Image.from_numpy(img)
        dev.convolve_separable(k, k, zb.BorderMode.REPLICATE, out=dev)
        assert np.array_equal(dev.to_numpy(), zo.conv_separable(img, k, k, "replicate"))


@pytest.mark.parametrize("shape,dtype", [((37, 53), np.uint8), ((31, 47, 3), np.uint8), ((40, 41, 4), np.uint8), ((37, 53), np.float32)])
@pytest.mark.parametrize("border", BORDERS)
def test_dense_convolve_bit_exact(zb, shape, dtype, border):
    rng = np.random.default_rng(abs(hash((shape, border))) % 2**32)
    for kh, kw in [(3, 3), (5, 3), (1, 7), (4, 4), (15, 15)]:
        img = rand_image(rng, shape, dtype)
        k = rng.standard_normal((kh, kw)).astype(np.float32) / (kh * kw)
        got = zb.Image.from_numpy(img).convolve(k, border_enum(zb, border)).to_numpy()
        assert np.array_equal(got, zo.convolve(img, k, border)), (kh, kw)


def test_reference_kats_through_the_gpu(zb):
    ident = np.zeros((3, 3), np.float32)
    ident[1, 1] = 1
    rng = np.random.default_rng(9)
    for shape in [(5, 5), (7, 9, 3), (6, 8, 4)]:  # filters.zig:370-398, :662-699
        img = rand_image(rng, shape, np.uint8)
        assert np.array_equal(zb.Image.from_numpy(img).convolve(ident, zb.BorderMode.ZERO).to_numpy(), img)
    img = np.full((5, 5, 3), 255, np.uint8)  # filters.zig:571-600
    out = zb.Image.from_numpy(img).convolve(np.full((3, 3), 1 / 9, np.float32), zb.BorderMode.ZERO).to_numpy()
    assert abs(int(out[0, 0, 0]) - 113) <= 1
    img = np.ones((10, 20), np.uint8)  # filters.zig:1302-1342
    k = np.array([[1, 1, 1], [1, 0, 1], [1, 1, 1]], np.float32)
    out = zb.Image.from_numpy(img).convolve(k, zb.BorderMode.ZERO).to_numpy()
    assert np.all(out[1:9, 0] == 5) and np.all(out[1:9, 1] == 8)
    img = np.zeros((7, 7), np.float32)  # filters.zig:469-491
    img[3, 3] = 1
    out = zb.Image.from_numpy(img).convolve_separable([0.25, 0.5, 0.25], [0.25, 0.5, 0.25], zb.BorderMode.ZERO).to_numpy()
    assert out[3, 3] == np.float32(0.25) and out[3, 2] == np.float32(0.125)
    img = rand_image(rng, (9, 9, 4), np.uint8)  # filters.zig:1159-1180: sigma == 0 is a copy
    assert np.array_equal(zb.Image.from_numpy(img).gaussian_blur(0.0).to_numpy(), img)
    with pytest.raises(zb.ZignalError) as e:
        zb.Image.from_numpy(img).gaussian_blur(-1.0)
    assert e.value.name == "InvalidSigma"


@pytest.mark.parametrize("shape,dtype", FORMATS)
def test_gaussian_blur_matches_oracle(zb, shape, dtype):
    rng = np.random.default_rng(10)
    img = rand_image(rng, shape, dtype)
    for sigma in (0.5, 1.0, 2.25, 4.0):
        got = zb.Image.from_numpy(img).gaussian_blur(sigma).to_numpy()
        want = zo.gaussian_blur(img, sigma)
        if dtype == np.uint8:
            assert np.array_equal(got, want), sigma
        else:
            assert rel_err(got, want) <= TOL_F32, sigma


def test_host_twins_with_strided_views_and_sentinels(zb):
    rng = np.random.default_rng(11)
    base = rand_image(rng, (40, 50, 4), np.uint8)
    src = base[3:33, 4:44]                      # strided host view
    outbuf = np.full((44, 60, 4), 0xAA, np.uint8)
    dst = outbuf[5:35, 6:46]
    taps = zb.gaussian_taps(1.4)
    zb.host_conv_separable(src, taps, taps, zb.BorderMode.MIRROR, out=dst)
    assert np.array_equal(dst, zo.conv_separable(np.ascontiguousarray(src), taps, taps, "mirror"))
    mask = np.ones(outbuf.shape[:2], bool)
    mask[5:35, 6:46] = False
    assert np.all(outbuf[mask] == 0xAA)
    imgf = rand_image(rng, (70, 90, 4), np.float32)
    got = zb.host_gaussian_blur(imgf, 2.25)
    assert rel_err(got, zo.gaussian_blur(imgf, 2.25)) <= TOL_F32
    k = rng.standard_normal((3, 3)).astype(np.float32)
    assert np.array_equal(zb.host_convolve(src, k, zb.BorderMode.WRAP), zo.convolve(np.ascontiguousarray(src), k, "wrap"))


@pytest.mark.parametrize("dtype,shape", [(np.float32, (2200, 1024, 4)), (np.uint8, (4200, 2048, 4))])
@pytest.mark.parametrize("border", ["zero", "replicate", "mirror", "wrap"])
def test_host_pipeline_matches_device_path(zb, dtype, shape, border):
    """The pipelined host-pointer path (PCIe row bands overlapped with the kernel) must be bit-identical to the device-resident
    call on the same image, for ragged band counts, strided host views and every border mode (wrap takes the one-shot path)."""
    L = zb.lib()
    rng = np.random.default_rng(5)
    base = rand_image(rng, (shape[0], shape[1] + 8, 4), dtype)
    src = base[:, 3:3 + shape[1]]                                   # strided host view, >= 32 MiB so the pipeline engages
    taps = zb.gaussian_taps(2.4)
    bm = getattr(zb.BorderMode, border.upper())
    want = zb.Image.from_numpy(np.ascontiguousarray(src)).convolve_separable(taps, taps, bm).to_numpy()
    for band in (256, 320, 0):
        assert L.zb_tune(b"host.band_rows", band) == 0
        try:
            out = np.full_like(base, 7)
            dst = out[:, 5:5 + shape[1]]
            zb.host_conv_separable(src, taps, taps, bm, out=dst)
        finally:
            L.zb_tune(b"host.band_rows", 256)
        assert np.array_equal(dst, want), (band, border)
        assert np.all(out[:, :5] == 7) and np.all(out[:, 5 + shape[1]:] == 7)
    if border == "mirror":
        got = zb.host_gaussian_blur(np.ascontiguousarray(src), 2.4)
        assert np.array_equal(got, want)


@pytest.mark.parametrize("dtype,shape", [(np.float32, (300, 264, 4)), (np.uint8, (300, 300, 4)), (np.uint8, (90, 70, 3)), (np.float32, (64, 40))])
def test_conv_separable_rows_windows(zb, dtype, shape):
    """zb_conv_separable_rows (the sharding extension): any tiling of the output rows into windows reproduces the full call
    bit for bit, for the fused kernels and for the two-pass path (which convolves into scratch and keeps the window)."""
    import ctypes as C
    import torch
    from zignal_b200.image import _fptr, current_stream
    L = zb.lib()
    rng = np.random.default_rng(21)
    img = rand_image(rng, shape, dtype)
    taps = zb.gaussian_taps(2.25)
    src = zb.Image.from_numpy(img)
    for border in (zb.BorderMode.MIRROR, zb.BorderMode.ZERO, zb.BorderMode.WRAP):
        want = src.convolve_separable(taps, taps, border).to_numpy()
        out = zb.Image.from_numpy(np.zeros_like(img))
        a, d = src._zb(), out._zb()
        cuts = sorted({0, 7, 8, shape[0] // 2, shape[0] - 7, shape[0]})
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            zb._ffi.check(L.zb_conv_separable_rows(a, d, int(src.pixfmt), _fptr(taps), taps.size, _fptr(taps), taps.size, int(border),
                                                   C.c_uint32(r0), C.c_uint32(0 if r1 == shape[0] else r1), current_stream()))
        torch.cuda.synchronize()
        assert np.array_equal(out.to_numpy(), want), border
    assert L.zb_conv_separable_rows(a, a, int(src.pixfmt), _fptr(taps), taps.size, _fptr(taps), taps.size, 2, 0, 0, None) != 0  # in place: refused


def test_row_block_conv_single_rank(zb):
    """RowBlock.conv_separable with one rank is the plain call on the interior (and wrap goes through the local halo copy)."""
    import torch
    from zignal_b200 import shard
    rng = np.random.default_rng(8)
    img = rand_image(rng, (96, 264, 4), np.float32)
    taps = zb.gaussian_taps(2.25)
    for halo in (0, 8):
        for border in (zb.BorderMode.MIRROR, zb.BorderMode.WRAP, zb.BorderMode.ZERO):
            sb = shard.RowBlock(96, 264, zb.PixFmt.RGBAF32, halo, "cuda", 0, 1)
            ob = shard.RowBlock(96, 264, zb.PixFmt.RGBAF32, halo, "cuda", 0, 1)
            sb.interior_tensor().copy_(torch.from_numpy(img).cuda())
            sb.conv_separable(ob, taps, taps, border)
            torch.cuda.synchronize()
            want = zb.Image.from_numpy(img).convolve_separable(taps, taps, border).to_numpy()
            assert np.array_equal(ob.interior_tensor().cpu().numpy(), want), (halo, border)


@pytest.mark.parametrize("shape", [(400, 1500), (330, 800, 3), (300, 1501), (260, 699, 3), (280, 516, 4)])
def test_tile_u8_kernel_interior_tiles(zb, shape):
    """Images large enough to have interior tiles (which the tile kernels copy as 32-bit words when base, pitch and row length are
    4-byte aligned; the odd widths keep the per-byte loader): Gaussian taps (dot-product variant) and signed taps (IMAD variant),
    a view whose rows start at an odd byte, bit-exact against the oracle."""
    L = zb.lib()
    rng = np.random.default_rng(shape[1])
    img = rand_image(rng, shape, np.uint8)
    dev = zb.Image.from_numpy(img)
    for k in (zb.gaussian_taps(2.25), zb.gaussian_taps(1.0), (rng.standard_normal(9) * 0.4).astype(np.float32)):
        for border in ("mirror", "zero"):
            if len(shape) == 3 and shape[2] == 4:
                L.zb_set_force_generic(0)
            got = dev.convolve_separable(k, k, border_enum(zb, border)).to_numpy()
            name = L.zb_last_kernel().decode()
            assert name.startswith("sep_tile_u8") or name.startswith("fused_sep_rgba8"), name
            assert np.array_equal(got, zo.conv_separable(img, k, k, border)), (name, border)
    v = dev.view(zb.Rectangle(3, 2, shape[1] - 5, shape[0] - 1))
    crop = np.ascontiguousarray(img[2:shape[0] - 1, 3:shape[1] - 5])
    got = v.convolve_separable(zb.gaussian_taps(2.25), zb.gaussian_taps(2.25), zb.BorderMode.REPLICATE).to_numpy()
    assert L.zb_last_kernel().decode().startswith("sep_tile_u8")
    assert np.array_equal(got, zo.conv_separable(crop, zb.gaussian_taps(2.25), zb.gaussian_taps(2.25), "replicate"))


@pytest.mark.parametrize("shape", [(70, 131), (129, 257, 3), (200, 90, 3), (65, 300, 4), (33, 1000)])
@pytest.mark.parametrize("border", BORDERS)
def test_tile_u8_kernel_against_oracle_and_two_pass(zb, shape, border):
    """The single-pass tile kernel for 8-bit images of any channel count / alignment: odd and even tap counts, different x / y
    kernels, every border mode, strided views -- bit-identical to the oracle and to the two-pass path."""
    L = zb.lib()
    rng = np.random.default_rng(shape[0] + shape[1])
    img = rand_image(rng, shape, np.uint8)
    dev = zb.Image.from_numpy(img)
    bm = border_enum(zb, border)
    for nx, ny in [(3, 3), (15, 15), (4, 9), (1, 7), (31, 2), (5, 29)]:
        kx, ky = _taps(rng, nx), _taps(rng, ny)
        want = zo.conv_separable(img, kx, ky, border)
        for dp in (1, 0):   # dot-product variant (byte taps, half <= 8) and the IMAD variant: one result
            L.zb_tune(b"conv.u8_dp", dp)
            got = dev.convolve_separable(kx, ky, bm).to_numpy()
            name = L.zb_last_kernel().decode()
            L.zb_tune(b"conv.u8_dp", 1)
            assert name in ("sep_tile_u8", "sep_tile_u8_dp") or (name.startswith("fused_sep_rgba8") and len(shape) == 3 and shape[2] == 4), (nx, ny, name)
            if name.startswith("sep_tile"):
                assert (name == "sep_tile_u8_dp") == bool(dp and max(nx, ny) // 2 <= 8 and max(nx, ny) // 2 >= 1 and _dp_eligible(kx, ky)), (nx, ny, name, dp)
            assert np.array_equal(got, want), (nx, ny, dp, name)
    L.zb_set_force_generic(1)
    try:
        kx, ky = _taps(rng, 11), _taps(rng, 7)
        two_pass = dev.convolve_separable(kx, ky, bm).to_numpy()
    finally:
        L.zb_set_force_generic(0)
    assert np.array_equal(dev.convolve_separable(kx, ky, bm).to_numpy(), two_pass)
    # strided source and destination views
    v = dev.view(zb.Rectangle(2, 3, shape[1] - 3, shape[0] - 1))
    out = zb.Image.from_numpy(np.full(shape, 5, np.uint8))
    ov = out.view(zb.Rectangle(2, 3, shape[1] - 3, shape[0] - 1))
    v.convolve_separable(kx, ky, bm, out=ov)
    res = out.to_numpy()
    assert np.array_equal(res[3:shape[0] - 1, 2:shape[1] - 3], zo.conv_separable(np.ascontiguousarray(img[3:shape[0] - 1, 2:shape[1] - 3]), kx, ky, border))
    res[3:shape[0] - 1, 2:shape[1] - 3] = 5
    assert np.all(res == 5)


def test_golden_fixtures(zb):
    g = golden()
    L = zb.lib()
    for name, case in g["conv"].items():
        rng = np.random.default_rng(case["seed"])
        dtype = np.uint8 if case["dtype"] == "u8" else np.float32
        img = rand_image(rng, tuple(case["shape"]), dtype)
        taps = zb.gaussian_taps(case["sigma"])
        L.zb_set_exact_f32(1)
        got = zb.Image.from_numpy(img).gaussian_blur(case["sigma"]).to_numpy()
        L.zb_set_exact_f32(0)
        assert sha(img) == case["input_sha256"], name
        assert sha(got) == case["output_sha256"], name


def test_full_size_c2_properties(zb):
    """BASELINE config 2: 15x15 Gaussian on 8192x8192 RGBA f32.  The oracle would need minutes for the whole
    image, so full size is checked through size-independent properties: a row band cropped with its halo must
    equal the oracle on that band (interior rows are independent of the rest), image borders likewise, and a
    constant image must stay constant."""
    import torch
    R = C = 8192
    gen = torch.Generator(device="cuda").manual_seed(2)
    x = torch.rand(R, C, 4, device="cuda", dtype=torch.float32, generator=gen)
    src = zb.Image.from_tensor(x)
    taps = zb.gaussian_taps(2.25)
    assert taps.size == 15
    out = src.gaussian_blur(2.25).tensor()
    assert zb.lib().zb_last_kernel().decode() == "fused_sep_rgbaf32"
    for (r0, r1, c0, c1) in [(0, 40, 0, 600), (4000, 4060, 3800, 4500), (R - 40, R, C - 600, C), (250, 270, 0, C)]:
        # halo of 7 around the window, clipped at the image border (where the mirror rule then matches the oracle's)
        hr0, hr1, hc0, hc1 = max(r0 - 7, 0), min(r1 + 7, R), max(c0 - 7, 0), min(c1 + 7, C)
        crop = x[hr0:hr1, hc0:hc1].cpu().numpy()
        want = zo.conv_separable(crop, taps, taps, "mirror")
        a, b = r0 - hr0, c0 - hc0
        # only compare pixels whose support lies in the crop or at a true image border
        sub_w = want[a:a + (r1 - r0), b:b + (c1 - c0)]
        sub_g = out[r0:r1, c0:c1].cpu().numpy()
        assert rel_err(sub_g, sub_w) <= TOL_F32, (r0, c0)
    const = torch.full((R, C, 4), 0.625, device="cuda", dtype=torch.float32)
    oc = zb.Image.from_tensor(const).gaussian_blur(2.25).tensor()
    assert float((oc - 0.625).abs().max()) <= 0.625 * 1e-5
