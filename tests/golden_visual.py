"""Seeded inputs and the case table of the diff / applyColormap / flip / invert fixtures, shared by the generator
(tests/golden/make_golden_visual.py), the CPU tests of the oracle (tests/test_visual_host.py) and the GPU tests (tests/test_gpu_visual.py).
Every image comes from numpy's PCG64, so the fixtures only pin the oracle's output."""
import numpy as np

import visual_oracle as zo

FORMATS = ("u8", "f32", "rgb8", "rgba8", "rgbaf32")
PIX = {"u8": 0, "f32": 1, "rgb8": 2, "rgba8": 3, "rgbaf32": 4}
_SHAPE = {"u8": (), "f32": (), "rgb8": (3,), "rgba8": (4,), "rgbaf32": (4,)}


def random_image(fmt, rows, cols, seed, specials=False):
    """Integers over 0..255, or floats over [-0.25, 1.25); with specials, floats also hold NaN, +inf, -inf and -0.0."""
    rng = np.random.default_rng(seed)
    shape = (rows, cols) + _SHAPE[fmt]
    if fmt not in ("f32", "rgbaf32"):
        return rng.integers(0, 256, shape, dtype=np.uint8)
    img = (rng.random(shape, dtype=np.float32) * np.float32(1.5) - np.float32(0.25)).astype(np.float32)
    if specials and img.size:
        flat = img.reshape(-1)
        idx = rng.choice(flat.size, size=max(4, flat.size // 50), replace=flat.size < 4)
        flat[idx] = rng.choice(np.array([np.nan, np.inf, -np.inf, -0.0], np.float32), size=idx.size)
    return img


def near_pair(fmt, rows, cols, seed):
    """A second image that differs from the first by small amounts (mostly 0..3 per component), so thresholds matter."""
    a = random_image(fmt, rows, cols, seed)
    rng = np.random.default_rng(seed + 1)
    if a.dtype == np.uint8:
        b = np.clip(a.astype(np.int16) + rng.integers(-3, 4, a.shape), 0, 255).astype(np.uint8)
    else:
        b = (a + rng.integers(-3, 4, a.shape).astype(np.float32) * np.float32(0.125)).astype(np.float32)
    return a, b


# name -> (op, fmt, rows, cols, seed, params)
CASES = {
    "diff_rgba8_cli_t2": ("diff", "rgba8", 97, 131, 1, dict(threshold=2.0, scale=1.0, binary=False, force_opaque=True)),
    "diff_rgba8_binary": ("diff", "rgba8", 64, 65, 2, dict(threshold=1.0, scale=1.0, binary=True, force_opaque=False)),
    "diff_u8_scale_neg": ("diff", "u8", 33, 257, 3, dict(threshold=0.0, scale=-1.5, binary=False, force_opaque=False)),
    "diff_rgb8_scale40": ("diff", "rgb8", 50, 77, 4, dict(threshold=0.0, scale=40.0, binary=False, force_opaque=False)),
    "diff_f32_scale3": ("diff", "f32", 41, 129, 5, dict(threshold=0.25, scale=3.0, binary=False, force_opaque=False)),
    "diff_rgbaf32_opaque": ("diff", "rgbaf32", 29, 61, 6, dict(threshold=0.125, scale=2.0, binary=False, force_opaque=True)),
    "colormap_u8_jet_auto": ("colormap", "u8", 60, 90, 7, dict(map=zo.JET, min=None, max=None)),
    "colormap_f32_turbo_partial": ("colormap", "f32", 45, 70, 8, dict(map=zo.TURBO, min=0.1, max=None)),
    "colormap_rgb8_viridis_range": ("colormap", "rgb8", 31, 47, 9, dict(map=zo.VIRIDIS, min=0.2, max=0.8)),
    "colormap_rgbaf32_inferno_auto": ("colormap", "rgbaf32", 23, 53, 10, dict(map=zo.INFERNO, min=None, max=None)),
    "colormap_rgba8_heat_auto": ("colormap", "rgba8", 37, 41, 11, dict(map=zo.HEAT, min=None, max=100.0)),
    "flip_lr_rgb8_odd": ("flip_lr", "rgb8", 17, 33, 12, {}),
    "flip_tb_rgbaf32_odd": ("flip_tb", "rgbaf32", 19, 8, 13, {}),
    "invert_rgba8": ("invert", "rgba8", 21, 35, 14, {}),
    "invert_rgbaf32": ("invert", "rgbaf32", 21, 35, 15, {}),
}


def case_inputs(name):
    op, fmt, rows, cols, seed, _ = CASES[name]
    if op == "diff":
        return near_pair(fmt, rows, cols, seed)
    return (random_image(fmt, rows, cols, seed),)


def run_case(name):
    """The oracle's outputs of a case: {'out': array[, 'stats': dict]}."""
    op, fmt, rows, cols, seed, prm = CASES[name]
    inputs = case_inputs(name)
    if op == "diff":
        out, stats = zo.diff(inputs[0], inputs[1], **prm)
        return {"out": out, "stats": stats}
    img = inputs[0].copy()
    if op == "colormap":
        return {"out": zo.apply_colormap(img, zo.colormap_lut(prm["map"]), prm["min"], prm["max"])}
    fn = {"flip_lr": zo.flip_left_right, "flip_tb": zo.flip_top_bottom, "invert": zo.invert}[op]
    return {"out": fn(img)}
