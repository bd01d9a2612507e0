"""Seeded inputs and the case table of the JPEG encoder fixtures, shared by the generator (tests/golden/make_golden_jpeg.py), the CPU tests
of the oracle (tests/test_jpeg_host.py) and the GPU tests (tests/test_gpu_jpeg.py).  Every image comes from numpy's PCG64 or a closed
formula, so the fixtures only pin the oracle's output."""
import numpy as np

FORMATS = ("u8", "f32", "rgb8", "rgba8", "rgbaf32")
PIX = {"u8": 0, "f32": 1, "rgb8": 2, "rgba8": 3, "rgbaf32": 4}
_SHAPE = {"u8": (), "f32": (), "rgb8": (3,), "rgba8": (4,), "rgbaf32": (4,)}


def noise(fmt, rows, cols, seed):
    """Integers over 0..255, or floats over [-0.25, 1.25) (so Image.convert's clamp is exercised).  NaN and other
    special values are tested in test_gpu_nonfinite.py."""
    rng = np.random.default_rng(seed)
    shape = (rows, cols) + _SHAPE[fmt]
    if fmt in ("f32", "rgbaf32"):
        return (rng.random(shape, dtype=np.float32) * np.float32(1.5) - np.float32(0.25)).astype(np.float32)
    return rng.integers(0, 256, shape, dtype=np.uint8)


def smooth(fmt, rows, cols, seed):
    """Gradients plus a little noise: the content of a photograph more than noise is."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:rows, 0:cols].astype(np.float64)
    planes = [127 + 100 * np.sin(x / 9.0 + k) * np.cos(y / 13.0 - k) + rng.normal(0, 6, (rows, cols)) for k in range(4)]
    v = np.clip(np.stack(planes, -1), 0, 255)
    if fmt == "u8":
        return v[..., 0].astype(np.uint8)
    if fmt == "f32":
        return (v[..., 0] / 255).astype(np.float32)
    if fmt == "rgb8":
        return v[..., :3].astype(np.uint8)
    if fmt == "rgba8":
        return v.astype(np.uint8)
    return (v / 255).astype(np.float32)


def dc_ramp(rows, cols):
    """Rgb(u8) blocks alternating between black and white in a checker of whole 8x8 blocks: at quality 100 the DC divisor is 1 and every
    DC difference is about +-2040, category 11."""
    y, x = np.mgrid[0:rows, 0:cols]
    v = np.where(((y // 8) + (x // 8)) % 2 == 0, 0, 255).astype(np.uint8)
    return np.stack([v, v, v], -1)


def checkerboard(rows, cols):
    """One-pixel checkerboard: the largest AC magnitudes the FDCT can produce (coefficient (7, 7) of every block)."""
    y, x = np.mgrid[0:rows, 0:cols]
    v = np.where((y + x) % 2 == 0, 0, 255).astype(np.uint8)
    return np.stack([v, 255 - v, v], -1)


def trailing_runs(rows, cols, seed):
    """u8 blocks of flat grey with one random 8x8 basis pattern each; with quality 50 the last nonzero coefficient of the blocks lands at
    every zigzag index, 15, 31, 47 and 63 included (the trailing-ZRL rule of encodeBlock)."""
    rng = np.random.default_rng(seed)
    out = np.empty((rows, cols), np.uint8)
    yy, xx = np.mgrid[0:8, 0:8]
    for by in range(0, rows, 8):
        for bx in range(0, cols, 8):
            u, v = rng.integers(0, 8, 2)
            amp = rng.uniform(4, 120)
            blk = 128 + amp * np.cos((2 * xx + 1) * u * np.pi / 16) * np.cos((2 * yy + 1) * v * np.pi / 16) + rng.normal(0, 1.0, (8, 8))
            out[by:by + 8, bx:bx + 8] = np.clip(blk, 0, 255)[:rows - by, :cols - bx]
    return out


def make(kind, fmt, rows, cols, seed):
    if kind == "noise":
        return noise(fmt, rows, cols, seed)
    if kind == "smooth":
        return smooth(fmt, rows, cols, seed)
    if kind == "const0":
        return np.zeros((rows, cols) + _SHAPE[fmt], noise(fmt, 1, 1, 0).dtype)
    if kind == "const255":
        a = np.full((rows, cols) + _SHAPE[fmt], 255, np.uint8)
        return a if fmt not in ("f32", "rgbaf32") else np.ones(a.shape, np.float32)
    if kind == "dc_ramp":
        return dc_ramp(rows, cols)
    if kind == "checker":
        return checkerboard(rows, cols)
    if kind == "trailing":
        return trailing_runs(rows, cols, seed)
    raise ValueError(kind)


# name -> (kind, fmt, rows, cols, seed, quality, subsampling, density_dpi, comment)
CASES = {
    "rgb8_420_q90_smooth": ("smooth", "rgb8", 96, 128, 1, 90, 2, 72, None),
    "rgb8_444_q100_noise": ("noise", "rgb8", 37, 53, 2, 100, 0, 72, None),
    "rgb8_422_q50_smooth": ("smooth", "rgb8", 19, 25, 3, 50, 1, 300, b"zignal"),
    "u8_q85_smooth": ("smooth", "u8", 64, 48, 4, 85, 2, 72, b""),
    "u8_q1_noise": ("noise", "u8", 17, 33, 5, 1, 0, 96, None),
    "f32_420_q90_noise": ("noise", "f32", 33, 40, 6, 90, 2, 72, None),
    "rgba8_444_q85_smooth": ("smooth", "rgba8", 45, 80, 7, 85, 0, 72, None),
    "rgbaf32_420_q99_smooth": ("smooth", "rgbaf32", 31, 29, 8, 99, 2, 72, None),
    "rgb8_420_q100_dc_ramp": ("dc_ramp", "rgb8", 64, 64, 0, 100, 2, 72, None),
    "rgb8_444_q100_checker": ("checker", "rgb8", 24, 40, 0, 100, 0, 72, None),
    "u8_q50_trailing": ("trailing", "u8", 128, 128, 9, 50, 0, 72, None),
    "rgb8_1x1_q90": ("noise", "rgb8", 1, 1, 10, 90, 2, 72, None),
}


def case_input(name):
    kind, fmt, rows, cols, seed = CASES[name][:5]
    return make(kind, fmt, rows, cols, seed)


def case_options(name):
    quality, subsampling, density_dpi, comment = CASES[name][5:]
    return dict(quality=quality, subsampling=subsampling, density_dpi=density_dpi, comment=comment)
