"""Seeded HoughTransform cases shared by the fixture generator (tests/golden/make_golden_hough.py), the CPU regression test of the oracle
(tests/test_hough_host.py) and the GPU fixture test (tests/test_gpu_hough.py).  Each case builds a u8 edge map from numpy's PCG64 and names
the box, the Hough size and the findLines arguments; the accumulator starts at zero, as in the reference's example
(examples/src/hough_animation.zig:82-118)."""
import numpy as np

import hough_oracle as zo


def draw_lines(rows, cols, segments, width=1, value=255):
    """u8 image with straight segments ((x0, y0, x1, y1), ...) of the given width."""
    img = np.zeros((rows, cols), np.uint8)
    half = width / 2.0
    pen = [(ox, oy) for oy in np.arange(-half, half + 1e-9, 0.5) for ox in np.arange(-half, half + 1e-9, 0.5) if ox * ox + oy * oy <= half * half]
    for x0, y0, x1, y1 in segments:
        s = np.linspace(0.0, 1.0, int(4 * max(abs(x1 - x0), abs(y1 - y0))) + 2)
        for ox, oy in pen:
            x = np.rint(x0 + s * (x1 - x0) + ox).astype(np.int64)
            y = np.rint(y0 + s * (y1 - y0) + oy).astype(np.int64)
            ok = (x >= 0) & (x < cols) & (y >= 0) & (y < rows)
            img[y[ok], x[ok]] = value
    return img


def random_edges(seed, rows, cols, density, low=1):
    """Sparse random edge map with values in [low, 255]."""
    rng = np.random.default_rng(seed)
    img = rng.integers(low, 256, (rows, cols), dtype=np.uint8)
    img[rng.random((rows, cols)) >= density] = 0
    return img


def example_frame():
    """The reference example's call shape: a 400 x 400 frame with one thick line (drawLine width 5)."""
    return draw_lines(400, 400, [(80.0, 310.0, 330.0, 90.0)], width=5)


def sparse_4096():
    """A 4096 x 4096 map of a dozen long segments over sparse noise (about 60 k edge pixels)."""
    rng = np.random.default_rng(7)
    img = random_edges(8, 4096, 4096, 0.002)
    segs = [tuple(rng.uniform(0, 4096, 4)) for _ in range(12)]
    return np.maximum(img, draw_lines(4096, 4096, segs, width=2))


# name -> (edge map builder, box (l, t, r, b), size, threshold (None: max // 2, as the example), angle_nms, radius_nms)
CASES = {
    "example_400_box50_size300": (example_frame, (50, 50, 350, 350), 300, None, 5.0, 5.0),
    "lines_257x311_size256": (lambda: draw_lines(257, 311, [(0, 40, 310, 60), (100, 0, 120, 256), (20, 240, 290, 10)]), (0, 0, 256, 256), 256, 40,
                              10.0, 5.0),
    "random_120x90_size101_partly_outside": (lambda: random_edges(11, 120, 90, 0.05), (40, 30, 141, 131), 101, 12, 3.0, 3.0),
    "random_64x64_size33_odd": (lambda: random_edges(12, 64, 64, 0.3), (5, 9, 38, 42), 33, 0, 4.0, 2.0),
    "sparse_4096x4096_size4096": (sparse_4096, (0, 0, 4096, 4096), 4096, 600, 2.0, 8.0),
}


def edges(name):
    return CASES[name][0]()


def threshold_of(name, acc):
    th = CASES[name][3]
    return max(1, int(acc.max()) // 2) if th is None else th


def lines_array(lines):
    """Line list -> (n, 7) float32 array (the score is exact in f32 below 2^24) for hashing and comparison."""
    return np.array([[a, r, s, x1, y1, x2, y2] for a, r, s, x1, y1, x2, y2 in lines], np.float64).astype(np.float32).reshape(-1, 7)


def oracle(name, img=None):
    """(accumulator, lines) of the oracle for a case."""
    img = edges(name) if img is None else img
    _, box, size, _, an, rn = CASES[name]
    acc = zo.compute(size, img, box, np.zeros((size, size), np.uint32))
    return acc, zo.find_lines(size, acc, threshold_of(name, acc), an, rn)


def device(zb, torch, name, img):
    """(accumulator, lines) of the device for a case, lines as tuples like the oracle's."""
    _, box, size, _, an, rn = CASES[name]
    h = zb.HoughTransform(size)
    acc = torch.zeros((size, size), dtype=torch.int32, device="cuda")
    h.compute(zb.Image.from_numpy(img), zb.Rectangle(*box), acc)
    acc_np = acc.cpu().numpy().view(np.uint32)
    lines = h.find_lines(acc, threshold_of(name, acc_np), an, rn)
    return acc_np, [(l.angle, l.radius, l.score, l.p1[0], l.p1[1], l.p2[0], l.p2[1]) for l in lines]
