"""Seeded Shen-Castan cases shared by the fixture generator (tests/golden/make_golden_shen_castan.py), the CPU regression test of the oracle
(tests/test_shen_castan_host.py) and the GPU fixture test (tests/test_gpu_shen_castan.py).  Each case builds its input from numpy's PCG64 and
names a preset of the reference (ShenCastan.zig:51-99); the oracle and the device mirror run the same options."""
import numpy as np

import shen_castan_oracle as zo


def smooth_noise(seed, rows, cols, channels=0, sigma=6.0):
    """Smooth blobs plus Gaussian noise, u8 (rows, cols[, channels])."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:rows, 0:cols].astype(np.float64)
    base = 128 + 90 * np.sin(xx / 13.0 + 0.3) * np.cos(yy / 19.0) + 40 * ((xx // 37 + yy // 29) % 2)
    shape = (rows, cols) + ((channels,) if channels else ())
    if channels:
        base = base[..., None] * np.linspace(0.6, 1.0, channels)[None, None, :]
    return np.clip(base + rng.normal(0, sigma, shape), 0, 255).astype(np.uint8)


def _f32(seed, rows, cols):
    return smooth_noise(seed, rows, cols).astype(np.float32) / np.float32(255.0)


# name -> (input builder, preset name)
CASES = {
    "gray_300x410_default": (lambda: smooth_noise(101, 300, 410), "default"),
    "gray_233x517_thin": (lambda: smooth_noise(102, 233, 517), "thin"),
    "gray_190x260_strong_only": (lambda: smooth_noise(103, 190, 260), "strong_only"),
    "rgb_257x333_heavy_smooth": (lambda: smooth_noise(104, 257, 333, 3), "heavy_smooth"),
    "rgba_200x301_high_noise": (lambda: smooth_noise(105, 200, 301, 4), "high_noise"),
    "f32_150x170_sensitive": (lambda: _f32(106, 150, 170), "sensitive"),
    "gray_4200x4200_low_noise": (lambda: smooth_noise(107, 4200, 4200), "low_noise"),   # summed-area tables beyond 2^24
}


def oracle(name, img):
    return zo.shen_castan(img, zo.PRESETS[CASES[name][1]])


def device(zb, name, img):
    o = zo.PRESETS[CASES[name][1]]
    return zb.Image.from_numpy(img).shen_castan(o.smooth, o.window_size, o.high_ratio, o.low_rel, o.hysteresis, o.use_nms).to_numpy()
