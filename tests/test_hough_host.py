"""HoughTransform on the CPU: the reference's two tests (image/hough.zig:259-285) against the oracle (oracle/zo_hough.cpp, bound in
tests/hough_oracle.py), an independent numpy restatement that must equal the oracle bit for bit (votes, line list and f32 geometry), facts
that do not depend on either, the host-decided errors of the C ABI (no device is touched), the C++ and Zig mirrors, and the golden fixtures.
"""
import ctypes as C
import json
import math
import shutil
import subprocess
import textwrap
from pathlib import Path

import numpy as np
import pytest

import hough_oracle as zo
from golden_hough import CASES, edges, lines_array, oracle, threshold_of
from gpu_utils import sha

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_hough.json"
F = np.float32
_libm = C.CDLL("libm.so.6")
_libm.cosf.argtypes = [C.c_float]
_libm.cosf.restype = C.c_float
_libm.sinf.argtypes = [C.c_float]
_libm.sinf.restype = C.c_float


# ---- numpy restatement of hough.zig ------------------------------------------------------------------------------------------------
def np_tables(size):
    even = size - size % 2
    cos_t = [math.trunc(65536.0 * math.cos(t * math.pi / even) / math.sqrt(2.0)) for t in range(size)]
    sin_t = [math.trunc(65536.0 * math.sin(t * math.pi / even) / math.sqrt(2.0)) for t in range(size)]
    return np.array(cos_t, np.int64), np.array(sin_t, np.int64)


def np_compute(size, img, box, acc):
    """compute (:75-139) with np.bincount in int64, added to a prior uint32 accumulator."""
    l, t, r, b = box
    even = size - size % 2
    cos_t, sin_t = np_tables(size)
    al, at, ar, ab = l, t, min(r, img.shape[1]), min(b, img.shape[0])
    out = acc.astype(np.int64)
    if al < ar and at < ab:
        ys, xs = np.nonzero(img[at:ab, al:ar])
        x_val = 2 * (xs.astype(np.int64) + al - l) - (size - 1)
        y_val = 2 * (ys.astype(np.int64) + at - t) - (size - 1)
        offset = int(round(65536 * even / 4.0))
        cols = np.arange(size, dtype=np.int64)
        counts = np.zeros(size * size, np.int64)
        for i in range(0, len(xs), 2048):
            rho = x_val[i:i + 2048, None] * cos_t[None, :] + y_val[i:i + 2048, None] * sin_t[None, :]
            assert np.abs(rho).max(initial=0) < 2 ** 31
            rr = ((rho >> 1) + (offset << 1)) >> 16
            ok = (rr >= 0) & (rr < size)
            counts += np.bincount((rr * size + cols[None, :])[ok], minlength=size * size)
        out += counts.reshape(size, size)
    return out.astype(np.uint32)


def _clip(p1x, p1y, p2x, p2y, size):
    t0, t1 = F(0), F(1)
    dx, dy = p2x - p1x, p2y - p1y
    p = [-dx, dx, -dy, dy]
    q = [p1x - F(0), F(size) - p1x, p1y - F(0), F(size) - p1y]
    for pi, qi in zip(p, q):
        if pi == 0:
            if qi < 0:
                return p1x, p1y, p2x, p2y
        else:
            r = F(qi / pi)
            if pi < 0:
                if r > t1:
                    return p1x, p1y, p2x, p2y
                if r > t0:
                    t0 = r
            else:
                if r < t0:
                    return p1x, p1y, p2x, p2y
                if r < t1:
                    t1 = r
    if t0 > t1:
        return p1x, p1y, p2x, p2y
    return F(p1x + t0 * dx), F(p1y + t0 * dy), F(p1x + t1 * dx), F(p1y + t1 * dy)


def np_find_lines(size, acc, threshold, an, rn):
    """findLines (:142-204): candidates in row-major order, stable sort by score, greedy NMS, f32 geometry (libm cosf / sinf)."""
    R, Cc = acc.shape
    if R < 3 or Cc < 3:
        return []
    a = acc.astype(np.int64)
    mid = a[1:-1, 1:-1]
    nb = np.max(np.stack([a[1 + dr:R - 1 + dr, 1 + dc:Cc - 1 + dc] for dr in (-1, 0, 1) for dc in (-1, 0, 1) if dr or dc]), axis=0)
    rows, cols = np.nonzero((mid >= threshold) & (nb <= mid))
    scores = mid[rows, cols]
    order = np.argsort(-scores, kind="stable")
    center, even, an, rn = F(size - 1) / F(2), F(size - size % 2), F(an), F(rn)
    kept = []
    for k in order:
        angle = F(180) * (F(cols[k] + 1) - center) / even
        radius = (F(rows[k] + 1) - center) * np.sqrt(F(2))
        if any((abs(ea - angle) < an and abs(er - radius) < rn) or ((F(180) - abs(ea - angle)) < an and abs(er + radius) < rn)
               for ea, er, *_ in kept):
            continue
        theta = (angle + F(90)) * F(np.pi) / F(180)
        cos_t, sin_t = F(_libm.cosf(theta)), F(_libm.sinf(theta))
        huge = F(size) * F(2)
        pcx, pcy = radius * cos_t, radius * sin_t
        p1x, p1y = center + pcx + (-sin_t) * huge, center + pcy + cos_t * huge
        p2x, p2y = center + pcx - (-sin_t) * huge, center + pcy - cos_t * huge
        kept.append((angle, radius, int(scores[k])) + _clip(p1x, p1y, p2x, p2y, size))
    return [(float(a), float(r), s, float(x1), float(y1), float(x2), float(y2)) for a, r, s, x1, y1, x2, y2 in kept]


# ---- the reference's tests (hough.zig:259-285) -------------------------------------------------------------------------------------
def test_reference_detect_horizontal_line():
    size = 64
    img = np.zeros((size, size), np.uint8)
    img[32, :] = 255
    acc = zo.compute(size, img, (0, 0, size, size), np.zeros((size, size), np.uint32))
    lines = zo.find_lines(size, acc, 30, 10.0, 5.0)
    assert len(lines) >= 1
    assert abs(lines[0][0] - 0.0) <= 2.0


def test_reference_invalid_size():
    for size in (0, 1):
        with pytest.raises(zo.OracleStatus) as e:
            zo.tables(size)
        assert e.value.status == 5


# ---- numpy restatement == oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", [2, 3, 4, 5, 31, 33, 300, 4096, 32768])
def test_tables_match_restatement(size):
    cos_o, sin_o = zo.tables(size)
    cos_n, sin_n = np_tables(size)
    assert np.array_equal(cos_o, cos_n) and np.array_equal(sin_o, sin_n)
    assert np.max(np.abs(cos_n) + np.abs(sin_n)) <= 65536   # the i32 bound of zb_hough.cu


def _boxes(size, rows, cols):
    return {"inside": (0, 0, size, size), "offset": (3, 2, 3 + size, 2 + size), "partly_outside": (cols // 2, rows // 3, cols // 2 + size, rows // 3 + size),
            "fully_outside": (cols + 5, 0, cols + 5 + size, size)}


@pytest.mark.parametrize("size", [2, 3, 4, 5, 31, 33, 300])
@pytest.mark.parametrize("where", ["inside", "offset", "partly_outside", "fully_outside"])
def test_restatement_matches_oracle(size, where):
    rng = np.random.default_rng(size * 7 + len(where))
    rows, cols = size + 11, size + 17
    img = rng.integers(1, 256, (rows, cols), dtype=np.uint8)
    img[rng.random((rows, cols)) >= (0.02 if size >= 300 else 0.3)] = 0
    box = _boxes(size, rows, cols)[where]
    prior = rng.integers(0, 1000, (size, size), dtype=np.uint32)   # the accumulator is added to, not overwritten
    acc_o = zo.compute(size, img, box, prior.copy())
    acc_n = np_compute(size, img, box, prior)
    assert np.array_equal(acc_o, acc_n)
    if where == "fully_outside":
        assert np.array_equal(acc_o, prior)
    votes = acc_o.astype(np.int64) - prior
    for th in (int(votes.max()) // 2 + 1000, int(acc_o.max()) - 3, 0):
        assert zo.find_lines(size, acc_o, th, 4.0, 3.0) == np_find_lines(size, acc_o, th, 4.0, 3.0), th


def test_strided_views_match_contiguous():
    size = 31
    rng = np.random.default_rng(5)
    big = rng.integers(0, 256, (60, 90), dtype=np.uint8)
    big[big < 200] = 0
    view = big[7:50, 11:70]
    acc_big = np.full((size + 4, size + 9), 7, np.uint32)
    acc_view = acc_big[2:2 + size, 3:3 + size]
    zo.compute(size, view, (4, 6, 4 + size, 6 + size), acc_view)
    want = np_compute(size, np.ascontiguousarray(view), (4, 6, 4 + size, 6 + size), np.full((size, size), 7, np.uint32))
    assert np.array_equal(acc_view, want)
    assert (acc_big[:2] == 7).all() and (acc_big[2 + size:] == 7).all() and (acc_big[:, :3] == 7).all() and (acc_big[:, 3 + size:] == 7).all()


def test_plateaus_give_several_candidates():
    size = 40
    acc = np.zeros((size, size), np.uint32)
    acc[10, 5:9] = 50          # a plateau of four equal cells: every one of them is a local maximum
    acc[25, 20] = 80
    lines_o = zo.find_lines(size, acc, 10, 0.5, 0.5)
    assert lines_o == np_find_lines(size, acc, 10, 0.5, 0.5)
    assert [l[2] for l in lines_o] == [80, 50, 50, 50, 50]
    # stable: equal scores keep the row-major scan order (columns ascending)
    assert [l[0] for l in lines_o[1:]] == sorted(l[0] for l in lines_o[1:])
    assert len(zo.find_lines(size, acc, 10, 20.0, 20.0)) == 2


def test_wrap_around_nms():
    size = 101
    acc = np.zeros((size, size), np.uint32)
    acc[20, 1] = 90            # angle near -90, radius r
    acc[80, 99] = 70           # angle near +90, radius -r: the same line, caught only by the 180 - da branch
    acc[50, 50] = 30
    lines = zo.find_lines(size, acc, 1, 5.0, 3.0)
    assert lines == np_find_lines(size, acc, 1, 5.0, 3.0)
    assert [l[2] for l in lines] == [90, 30]
    assert len(zo.find_lines(size, acc, 1, 1.0, 3.0)) == 3


def test_small_accumulators_give_no_lines():
    for shape in ((2, 10), (10, 2), (0, 0)):
        assert zo.find_lines(8, np.ones(shape, np.uint32), 0, 1.0, 1.0) == []
    # any accumulator shape: findLines only needs the handle's size for the geometry
    acc = np.zeros((5, 9), np.uint32)
    acc[2, 4] = 3
    assert zo.find_lines(8, acc, 1, 1.0, 1.0) == np_find_lines(8, acc, 1, 1.0, 1.0)


# ---- independent facts --------------------------------------------------------------------------------------------------------------
def test_vertical_line_gives_plus_minus_90():
    size = 256
    img = np.zeros((size, size), np.uint8)
    img[:, 100] = 255
    acc = zo.compute(size, img, (0, 0, size, size), np.zeros((size, size), np.uint32))
    # theta = 0 (column 0, angle -90 x (1 - 1/size)) holds the peak: all size pixels in one bin
    assert acc[:, 0].max() == acc.max() == size
    # findLines scans the interior only, so tilt the line by about one angle column (0.7 degrees): it must come out at about +-90
    tilted = np.zeros((size, size), np.uint8)
    rows = np.arange(size)
    tilted[rows, np.rint(100 - rows * math.tan(math.pi / size)).astype(int)] = 255   # normal at theta = pi / size: column 1
    acc = zo.compute(size, tilted, (0, 0, size, size), np.zeros((size, size), np.uint32))
    lines = zo.find_lines(size, acc, size // 2, 10.0, 5.0)
    assert lines and abs(abs(lines[0][0]) - 90.0) <= 2.0, lines[:3]


def test_vote_total_equals_brute_force_count():
    size = 31
    rng = np.random.default_rng(3)
    img = (rng.random((40, 35)) < 0.1).astype(np.uint8) * rng.integers(1, 256, (40, 35), dtype=np.uint8)
    box = (2, 5, 2 + size, 5 + size)
    acc = zo.compute(size, img, box, np.zeros((size, size), np.uint32))
    even = size - 1
    offset = 65536 * even // 4
    n = 0
    for r in range(5, min(5 + size, 40)):
        for c in range(2, min(2 + size, 35)):
            if img[r, c]:
                x, y = 2 * (c - 2) - (size - 1), 2 * (r - 5) - (size - 1)
                for t in range(size):
                    th = t * math.pi / even
                    rho = x * math.trunc(65536 * math.cos(th) / math.sqrt(2)) + y * math.trunc(65536 * math.sin(th) / math.sqrt(2))
                    n += 0 <= ((rho >> 1) + 2 * offset) >> 16 < size
    assert int(acc.sum()) == n > 0


# ---- host-decided errors of the C ABI (no device is touched) -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zbl():
    from zignal_b200 import _ffi
    return _ffi


def test_abi_create_errors(zbl):
    L = zbl.lib()
    h = C.c_void_p()
    assert L.zb_hough_create(0, None, None, C.byref(h)) == 5
    assert L.zb_hough_create(1, None, None, C.byref(h)) == 5
    assert L.zb_hough_create(32769, None, None, C.byref(h)) == 3
    assert L.zb_hough_create(64, None, None, None) == 5
    assert L.zb_hough_create(32768, None, None, C.byref(h)) == 0 and h.value
    assert L.zb_hough_destroy(h) == 0
    with pytest.raises(zbl.ZignalError) as e:
        import zignal_b200 as zb
        zb.HoughTransform(1)
    assert e.value.name == "InvalidArgument"


def test_abi_compute_and_find_lines_errors(zbl):
    L = zbl.lib()
    h = C.c_void_p()
    assert L.zb_hough_create(16, None, None, C.byref(h)) == 0
    try:
        dummy = C.c_void_p(0x1000)   # never dereferenced: every case below is rejected on the host
        e = zbl.ZbImage(dummy, 20, 20, 20)
        acc = zbl.ZbImage(dummy, 16, 16, 16)
        assert L.zb_hough_compute(None, e, 0, 0, 16, 16, acc, None) == 5
        assert L.zb_hough_compute(h, None, 0, 0, 16, 16, acc, None) == 5
        assert L.zb_hough_compute(h, e, 0, 0, 16, 16, None, None) == 5
        assert L.zb_hough_compute(h, e, 0, 0, 17, 16, acc, None) == 1    # box 17 x 16
        assert L.zb_hough_compute(h, e, 3, 0, 2, 16, acc, None) == 1     # r < l: width 0
        assert L.zb_hough_compute(h, e, 0, 0, 16, 16, zbl.ZbImage(dummy, 16, 15, 16), None) == 1
        assert L.zb_hough_compute(h, e, 0, 0, 16, 16, zbl.ZbImage(dummy, 15, 16, 16), None) == 1
        n = C.c_uint32(7)
        out = (zbl.ZbHoughLine * 4)()
        assert L.zb_hough_find_lines(None, acc, 1, 1.0, 1.0, out, 4, C.byref(n), None) == 5
        assert L.zb_hough_find_lines(h, None, 1, 1.0, 1.0, out, 4, C.byref(n), None) == 5
        assert L.zb_hough_find_lines(h, acc, 1, 1.0, 1.0, out, 4, None, None) == 5
        assert L.zb_hough_find_lines(h, acc, 1, 1.0, 1.0, None, 4, C.byref(n), None) == 5
        assert L.zb_hough_find_lines(h, zbl.ZbImage(dummy, 2, 50, 50), 1, 1.0, 1.0, out, 4, C.byref(n), None) == 0 and n.value == 0
    finally:
        L.zb_hough_destroy(h)


# ---- the C++ and Zig mirrors ---------------------------------------------------------------------------------------------------------
CPP = textwrap.dedent(r"""
    #include <cstdio>
    #include "zignal_b200/host/zignal.hpp"
    using namespace zignal;
    void instantiate() {                      // never called: type-checks the wrappers against the C ABI
        HoughTransform h(64);
        DeviceImage<uint8_t> e;
        DeviceImage<uint32_t> acc;
        h.compute(e, 0, 0, 64, 64, acc);
        std::vector<HoughTransform::Line> lines = h.findLines(acc, 10, 5.0f, 5.0f);
        (void)lines;
    }
    int main() {
        try { HoughTransform h(1); } catch (const Error& err) { std::printf("%d %s\n", err.status, err.what()); }
        try { HoughTransform h(40000); } catch (const Error& err) { std::printf("%d %s\n", err.status, err.what()); }
        HoughTransform ok(300);
        std::printf("%u %u\n", ok.size(), ok.evenSize());
        return 0;
    }
""")


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")
def test_cpp_mirror_hough(tmp_path):
    lib_dir = ROOT / "zignal_b200" / "lib"
    src = tmp_path / "hough.cpp"
    src.write_text(CPP)
    exe = tmp_path / "hough"
    gxx = "/usr/bin/g++" if Path("/usr/bin/g++").exists() else "g++"
    res = subprocess.run([gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT), str(src), "-o", str(exe), "-L", str(lib_dir),
                          "-lzignal_b200", f"-Wl,-rpath,{lib_dir}"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.strip().splitlines()
    assert lines[0].startswith("5 ") and "InvalidArgument" in lines[0]
    assert lines[1].startswith("3 ") and "Unsupported" in lines[1]
    assert lines[2] == "300 300"


def test_zig_shim_has_hough_transform():
    import re
    z = (ROOT / "zig" / "zignal_b200.zig").read_text()
    for pattern in (r"pub const HoughTransform = struct", r"pub const Line = struct", r"pub fn init\(allocator: Allocator, size: u32\)",
                    r"pub fn deinit\(self: \*Self\)", r"pub fn compute\(self: Self, edges: anytype, box: anytype, accumulator: anytype\)",
                    r"pub fn findLines\(\s*self: Self,\s*allocator: Allocator,\s*accumulator: anytype,\s*threshold: u32,\s*angle_nms_thresh: f32,\s*radius_nms_thresh: f32,?\s*\)",
                    r"pub const HoughLine = extern struct", r"pub const Hough = opaque"):
        assert re.search(pattern, z), pattern


# ---- golden fixtures -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_golden_fixtures_pin_the_oracle(name):
    want = json.loads(GOLDEN.read_text())["cases"][name]
    img = edges(name)
    assert sha(img) == want["input_sha256"]
    acc, lines = oracle(name, img)
    assert sha(acc) == want["accumulator_sha256"]
    assert len(lines) == want["lines"] and sha(lines_array(lines)) == want["lines_sha256"]
    if CASES[name][2] <= 300:
        _, box, size, _, an, rn = CASES[name]
        assert np.array_equal(acc, np_compute(size, img, box, np.zeros((size, size), np.uint32)))
        assert lines == np_find_lines(size, acc, threshold_of(name, acc), an, rn)
