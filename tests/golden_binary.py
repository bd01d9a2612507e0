"""Seeded cases of the 8-bit histogram family and binary morphology shared by the fixture generator (tests/golden/make_golden_binary.py),
the CPU regression test of the oracle (tests/test_binary_host.py) and the GPU fixture test (tests/test_gpu_binary.py).  Each case builds its
input from numpy's PCG64 and names the oracle call and the equivalent call on the device mirror; every listed operation is bit-exact."""
import numpy as np

import binary_oracle as zo
from gpu_utils import rand_image


def _img(seed, shape):
    return rand_image(np.random.default_rng(seed), shape, np.uint8)


def _smooth(seed, rows, cols):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:rows, 0:cols].astype(np.float64)
    base = 128 + 90 * np.sin(xx / 17.0) * np.cos(yy / 23.0) + rng.normal(0, 4.0, (rows, cols))
    return np.clip(base, 0, 255).astype(np.uint8)


CROSS = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], np.uint8)
ASYM3X5 = np.array([[1, 0, 0, 0, 0], [0, 0, 1, 0, 1], [0, 1, 0, 0, 1]], np.uint8)   # holes, not symmetric

# name -> (input builder, oracle call, device call).  Device calls take (zb, image array) and return a numpy array.
CASES = {
    "equalize_rgba": (lambda: _img(77, (110, 143, 4)), lambda a: zo.equalize(a), lambda zb, a: zb.Image.from_numpy(a).equalize().to_numpy()),
    "autocontrast_rgb_0.02": (lambda: (_img(78, (96, 131, 3)) // 3 + 40).astype(np.uint8), lambda a: zo.autocontrast(a, 0.02),
                              lambda zb, a: zb.Image.from_numpy(a).autocontrast(0.02).to_numpy()),
    "otsu_smooth_gray": (lambda: _smooth(79, 180, 250), lambda a: zo.threshold_otsu(a)[0],
                         lambda zb, a: zb.Image.from_numpy(a).threshold_otsu()[0].to_numpy()),
    # the QR detector's call (qrcode/detector.zig:74): radius max(min(rows, cols) / 16, 8), c = 4
    "adaptive_mean_1080p_r67_c4": (lambda: _smooth(80, 1080, 1920), lambda a: zo.threshold_adaptive_mean(a, 67, 4.0),
                                   lambda zb, a: zb.Image.from_numpy(a).threshold_adaptive_mean(67, 4.0).to_numpy()),
    "open_cross_x2": (lambda: _smooth(81, 140, 177) // 128 * 255, lambda a: zo.morph_binary(a, CROSS, 2, "open"),
                      lambda zb, a: zb.Image.from_numpy(a).open_binary(CROSS, 2).to_numpy()),
    "close_asym3x5": (lambda: (_img(82, (120, 161)) > 140).astype(np.uint8) * 255, lambda a: zo.morph_binary(a, ASYM3X5, 1, "close"),
                      lambda zb, a: zb.Image.from_numpy(a).close_binary(ASYM3X5, 1).to_numpy()),
}
