"""Seeded colour-quantization and dithering inputs and cases shared by the fixture generator (tests/golden/make_golden_quantize.py), the
CPU tests of the oracle (tests/test_quantize_host.py) and the GPU tests (tests/test_gpu_quantize.py).  Every image comes from numpy's
PCG64 or a closed form, so the fixtures only pin the oracle's output."""
import numpy as np

import quantize_oracle as zo

FORMATS = ("u8", "f32", "rgb8", "rgba8", "rgbaf32")
_SHAPE = {"u8": (), "f32": (), "rgb8": (3,), "rgba8": (4,), "rgbaf32": (4,)}
DITHER_MODES = (zo.NONE, zo.FLOYD_STEINBERG, zo.ATKINSON, zo.ORDERED, zo.AUTO)


def random_image(fmt, rows, cols, seed):
    rng = np.random.default_rng(seed)
    shape = (rows, cols) + _SHAPE[fmt]
    if fmt in ("f32", "rgbaf32"):
        return (rng.random(shape, dtype=np.float32) * np.float32(1.2) - np.float32(0.1)).astype(np.float32)   # some out of [0, 1]
    return rng.integers(0, 256, shape, dtype=np.uint8)


def smooth_rgb(rows, cols, seed=0):
    """A smooth colour field with mild noise: the kind of frame a GIF encoder dithers."""
    rng = np.random.default_rng(seed)
    rr, cc = np.mgrid[0:rows, 0:cols].astype(np.float64)
    r = 127.5 + 127.5 * np.sin(rr / max(rows, 1) * 3.1 + cc / max(cols, 1) * 1.3)
    g = 255.0 * cc / max(cols - 1, 1)
    b = 255.0 * rr / max(rows - 1, 1)
    img = np.stack([r, g, b], axis=2) + rng.normal(0, 6, (rows, cols, 3))
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def all_bins_shuffled(seed=0):
    """A 256 x 256 Rgb(u8) image touching all 32768 5-bit bins in shuffled order (each bin twice, low bits random)."""
    rng = np.random.default_rng(seed)
    keys = np.concatenate([rng.permutation(32768), rng.permutation(32768)])
    r5, g5, b5 = keys >> 10, (keys >> 5) & 31, keys & 31
    low = rng.integers(0, 8, (keys.size, 3))
    px = np.stack([(r5 << 3) | low[:, 0], (g5 << 3) | low[:, 1], (b5 << 3) | low[:, 2]], axis=1).astype(np.uint8)
    return px.reshape(256, 256, 3)


def random_palette(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 3), dtype=np.uint8)


def palette(kind, img=None):
    """'6x7x6', 'vga16', 'web216', 'adaptive<k>' or 'random<k>'."""
    if kind == "6x7x6":
        return zo.build_palette(None, zo.FIXED_6X7X6)
    if kind == "vga16":
        return zo.build_palette(None, zo.FIXED_VGA16)
    if kind == "web216":
        return zo.build_palette(None, zo.FIXED_WEB216)
    if kind.startswith("adaptive"):
        return zo.build_palette(img, zo.ADAPTIVE, int(kind[8:]))
    return random_palette(int(kind[6:]), 1000 + int(kind[6:]))


# name -> (image builder, palette kind, dither mode)
CASES = {
    "smooth_240x320_adaptive256_fs": (lambda: smooth_rgb(240, 320, 1), "adaptive256", zo.FLOYD_STEINBERG),
    "smooth_240x320_adaptive16_atkinson": (lambda: smooth_rgb(240, 320, 2), "adaptive16", zo.ATKINSON),
    "smooth_241x333_6x7x6_ordered": (lambda: smooth_rgb(241, 333, 3), "6x7x6", zo.ORDERED),
    "noise_97x131_vga16_fs": (lambda: random_image("rgb8", 97, 131, 4), "vga16", zo.FLOYD_STEINBERG),
    "noise_97x131_vga16_atkinson": (lambda: random_image("rgb8", 97, 131, 5), "vga16", zo.ATKINSON),
    "noise_64x65_web216_ordered": (lambda: random_image("rgb8", 64, 65, 6), "web216", zo.ORDERED),
    "all_bins_adaptive256_fs": (lambda: all_bins_shuffled(7), "adaptive256", zo.FLOYD_STEINBERG),
    "smooth_33x1000_random2_atkinson": (lambda: smooth_rgb(33, 1000, 8), "random2", zo.ATKINSON),
}


def run_chain(name, img=None):
    """(palette, lut, index map of the input, dithered image) of a case by the oracle."""
    builder, kind, mode = CASES[name]
    img = builder() if img is None else img
    pal = palette(kind, img)
    lut = zo.color_lut(pal)
    idx = zo.palette_lookup(img, lut)
    out = zo.dither(img.copy(), pal, lut, mode)
    return pal, lut, idx, out
