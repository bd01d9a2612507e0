"""CPU checks of Image.floodFill: the reference's own tests (image/tests/flood_fill.zig) against the oracle (oracle/zo_flood_fill.cpp), an
independent restatement that pins the oracle (scipy.ndimage.label for .seed, scipy.sparse.csgraph.connected_components for .neighbor) over
all five pixel formats, both connectivities and thresholds 0 / small / large / negative / NaN / inf with NaN, +-inf and -0.0 among the f32
inputs, the golden fixtures, the new status name, the argument errors the library decides before any device work, and the C++ mirror."""
import ctypes as C
import json
import shutil
import subprocess
import textwrap
from pathlib import Path

import numpy as np
import pytest
from scipy import ndimage, sparse
from scipy.sparse import csgraph

import flood_fill_oracle as zo
from golden_flood_fill import CASES, FORMATS, image, oracle, random_image, special_floats, spiral
from gpu_utils import sha

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_flood_fill.json"


# ---- the reference's tests (image/tests/flood_fill.zig) ---------------------------------------------------------------------------------

def test_reference_connectivity():
    img = np.zeros((5, 5), np.uint8)
    for r, c in ((0, 1), (1, 2), (2, 0), (2, 1), (2, 2), (2, 3), (2, 4), (3, 2), (4, 2)):
        img[r, c] = 5
    img4 = zo.flood_fill(img.copy(), 2, 2, 9, 0.0, 4)
    assert img4[0, 1] == 5 and img4[1, 2] == 9 and img4[2, 2] == 9
    img8 = zo.flood_fill(img.copy(), 2, 2, 9, 0.0, 8)
    assert img8[0, 1] == 9 and img8[1, 2] == 9 and img8[2, 2] == 9


def test_reference_threshold_modes():
    img = np.arange(5, dtype=np.uint8).reshape(1, 5)
    assert zo.flood_fill(img.copy(), 0, 0, 9, 1.0, 4, zo.SEED).tolist() == [[9, 9, 2, 3, 4]]
    assert zo.flood_fill(img.copy(), 0, 0, 9, 1.0, 4, zo.NEIGHBOR).tolist() == [[9, 9, 9, 9, 9]]


def test_reference_rgb():
    img = np.array([[[100, 100, 100], [100, 100, 103], [100, 100, 107]]], np.uint8)
    fill = [255, 0, 0]
    assert zo.flood_fill(img.copy(), 0, 0, fill, 4.0).tolist() == [[fill, fill, [100, 100, 107]]]
    assert zo.flood_fill(img.copy(), 0, 0, fill, 8.0).tolist() == [[fill, fill, fill]]


def test_reference_out_of_bounds():
    img = np.zeros((3, 3), np.uint8)
    with pytest.raises(zo.OracleStatus) as e:
        zo.flood_fill(img, 3, 3, 9, 1.0)
    assert e.value.status == zo.OUT_OF_BOUNDS
    assert not img.any()


# ---- an independent restatement ---------------------------------------------------------------------------------------------------------

def distance(a, b):
    """pixelDistance (flood_fill.zig:28-51) in f64, elementwise over two arrays of pixels: numpy rounds each operation separately."""
    a, b = np.asarray(a), np.asarray(b)
    if a.ndim == 2 or (a.ndim == 1 and b.ndim <= 1 and a.size == 1):
        return np.abs(a.astype(np.float64) - b.astype(np.float64))
    s = np.zeros(a.shape[:-1], np.float64)
    for ch in range(a.shape[-1]):
        d = a[..., ch].astype(np.float64) - b[..., ch].astype(np.float64)
        s = s + d * d
    return np.sqrt(s)


def restated(img, sr, sc, fill, threshold, connectivity, mode):
    """The filled image from a connected-component labelling of the edge graph (see zb_flood.cu for why it equals the reference's)."""
    rows, cols = img.shape[:2]
    with np.errstate(invalid="ignore"):
        if mode == zo.SEED:
            seed = img[sr, sc]
            mask = distance(img, np.broadcast_to(seed, img.shape)) <= threshold
            mask[sr, sc] = True
            structure = np.ones((3, 3), bool) if connectivity == 8 else ndimage.generate_binary_structure(2, 1)
            labels, _ = ndimage.label(mask, structure=structure)
            region = labels == labels[sr, sc]
        else:
            idx = np.arange(rows * cols).reshape(rows, cols)
            offsets = [(0, 1), (1, 0)] + ([(1, -1), (1, 1)] if connectivity == 8 else [])
            src, dst = [], []
            for dr, dc in offsets:
                r0, r1 = 0, rows - dr
                c0, c1 = max(0, -dc), cols - max(0, dc)
                if r1 <= r0 or c1 <= c0:
                    continue
                p = img[r0:r1, c0:c1]
                q = img[r0 + dr:r1 + dr, c0 + dc:c1 + dc]
                ok = distance(p, q) <= threshold
                src.append(idx[r0:r1, c0:c1][ok])
                dst.append(idx[r0 + dr:r1 + dr, c0 + dc:c1 + dc][ok])
            src = np.concatenate(src) if src else np.zeros(0, np.int64)
            dst = np.concatenate(dst) if dst else np.zeros(0, np.int64)
            g = sparse.coo_matrix((np.ones(src.size), (src, dst)), shape=(rows * cols, rows * cols))
            _, comp = csgraph.connected_components(g, directed=False)
            comp = comp.reshape(rows, cols)
            region = comp == comp[sr, sc]
    out = img.copy()
    out[region] = zo.fill_pixel(img, fill)
    return out


THRESHOLDS = {"zero": 0.0, "small": 0.3, "large": 200.0, "negative": -1.0, "nan": float("nan"), "inf": float("inf")}
FILLS = {"u8": 42, "f32": -7.25, "rgb8": (1, 2, 3), "rgba8": (9, 8, 7, 6), "rgbaf32": (0.5, -0.5, 2.0, np.nan)}


def _inputs(fmt, seed):
    rows, cols = (23, 37) if seed % 2 else (40, 17)
    img = random_image(fmt, rows, cols, seed, levels=2 + seed % 3)
    if fmt == "f32" and seed % 2:
        img = special_floats(rows, cols, seed)
    if fmt == "rgbaf32" and seed % 2:
        img = special_floats(rows, cols, seed, channels=4)
    return img


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("connectivity", [4, 8])
@pytest.mark.parametrize("mode", [zo.SEED, zo.NEIGHBOR], ids=["seed", "neighbor"])
def test_oracle_equals_component_labelling(fmt, connectivity, mode):
    scale = 1.0 if fmt in ("f32", "rgbaf32") else 255.0
    for seed in range(4):
        img = _inputs(fmt, seed)
        rng = np.random.default_rng(100 + seed)
        for name, th in THRESHOLDS.items():
            th = th * scale if name in ("small", "large") else th
            sr, sc = int(rng.integers(0, img.shape[0])), int(rng.integers(0, img.shape[1]))
            want = restated(img, sr, sc, FILLS[fmt], th, connectivity, mode)
            got = zo.flood_fill(img.copy(), sr, sc, FILLS[fmt], th, connectivity, mode)
            assert sha(got) == sha(want), (fmt, seed, name, sr, sc)


def test_oracle_equals_component_labelling_on_a_spiral():
    img = spiral(61)
    for conn in (4, 8):
        for mode in (zo.SEED, zo.NEIGHBOR):
            assert sha(zo.flood_fill(img.copy(), 0, 0, 1, 0.0, conn, mode)) == sha(restated(img, 0, 0, 1, 0.0, conn, mode))
    filled = zo.flood_fill(img.copy(), 0, 0, 1, 0.0, 4)
    assert (filled == 1).sum() == (img == 255).sum()          # one path: every path pixel is reached


def test_distance_is_symmetric_and_nan_is_never_within_threshold():
    rng = np.random.default_rng(0)
    a, b = special_floats(50, 50, 1, channels=4), special_floats(50, 50, 2, channels=4)
    with np.errstate(invalid="ignore"):
        da, db = distance(a, b), distance(b, a)
        assert np.array_equal(da, db, equal_nan=True)
        x = rng.integers(0, 256, (1000, 3)).astype(np.uint8)
        y = rng.integers(0, 256, (1000, 3)).astype(np.uint8)
        assert np.array_equal(distance(x, y), distance(y, x))
        assert not (np.float64(np.nan) <= np.inf)


# ---- golden fixtures --------------------------------------------------------------------------------------------------------------------

def test_golden_fixtures_match_the_oracle():
    gold = json.loads(GOLDEN.read_text())["cases"]
    assert set(gold) == set(CASES)
    for name in CASES:
        img = image(name)
        assert sha(img) == gold[name]["input_sha256"], name
        assert sha(oracle(name, img)) == gold[name]["output_sha256"], name


# ---- the C ABI: status name and argument errors (no device work) ------------------------------------------------------------------------

def test_out_of_bounds_status_name():
    import zignal_b200 as zb
    assert zb.lib().zb_status_name(27).decode() == "OutOfBounds"


def test_argument_errors_are_decided_before_the_device():
    import zignal_b200 as zb
    L = zb.lib()
    fake = C.c_void_p(0x1000)          # never dereferenced: every call below fails before any device work
    fill = np.zeros(16, np.uint8)
    fp = fill.ctypes.data_as(C.c_void_p)

    def call(rows=8, cols=8, fmt=0, r=0, c=0, f=fp, conn=4, mode=0, data=fake):
        img = zb.ZbImage(data, rows, cols, cols)
        return L.zb_flood_fill(C.byref(img), fmt, r, c, f, C.c_double(0.0), conn, mode, None)

    assert L.zb_flood_fill(None, 0, 0, 0, fp, C.c_double(0.0), 4, 0, None) == 5
    assert call(fmt=5) == 3 and call(fmt=-1) == 3
    assert call(conn=6) == 5 and call(conn=0) == 5
    assert call(mode=2) == 5 and call(mode=-1) == 5
    assert call(f=None) == 5
    assert call(r=8) == 27 and call(c=8) == 27 and call(r=2**32 - 1) == 27
    assert call(rows=0, cols=0) == 27 and call(rows=0, cols=5) == 27
    assert call(rows=65536, cols=65536) == 3 and call(rows=1 << 20, cols=1 << 12) == 3
    assert call(rows=65536, cols=65536, r=70000) == 27     # the reference's OutOfBounds comes first
    assert call(data=None) == 5


# ---- the C++ mirror ---------------------------------------------------------------------------------------------------------------------

PROGRAM = textwrap.dedent(r"""
    #include <cstdio>
    #include "zignal_b200/host/zignal.hpp"
    using namespace zignal;
    template <typename T> void instantiate(T v) {       // never called: type-checks floodFill against the C ABI for every pixel type
        DeviceImage<T> d;
        d.floodFill(1, 2, v);
        d.floodFill(1, 2, v, FloodFillOptions{2.5, FloodFillOptions::Connectivity::eight, FloodFillOptions::ThresholdMode::neighbor});
    }
    template void instantiate<uint8_t>(uint8_t);
    template void instantiate<float>(float);
    template void instantiate<Rgb8>(Rgb8);
    template void instantiate<Rgba8>(Rgba8);
    template void instantiate<RgbaF32>(RgbaF32);
    int main() {
        DeviceImage<uint8_t> d;
        d.rows = 3; d.cols = 3; d.stride = 3;
        d.data = reinterpret_cast<uint8_t*>(0x1000);   // OutOfBounds is decided before the device is touched
        try { d.floodFill(3, 0, 9); } catch (const Error& e) { std::printf("%d %s\n", e.status, e.what()); }
        return 0;
    }
""")


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")
def test_cpp_mirror_flood_fill(tmp_path):
    lib_dir = ROOT / "zignal_b200" / "lib"
    src = tmp_path / "flood.cpp"
    src.write_text(PROGRAM)
    exe = tmp_path / "flood"
    gxx = "/usr/bin/g++" if Path("/usr/bin/g++").exists() else "g++"
    res = subprocess.run([gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT), str(src), "-o", str(exe), "-L", str(lib_dir),
                          "-lzignal_b200", f"-Wl,-rpath,{lib_dir}"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert out.stdout.strip() == "27 zignal error.OutOfBounds"


def test_zig_mirror_has_flood_fill():
    zig = (ROOT / "zig" / "zignal_b200.zig").read_text()
    assert "pub fn floodFill(self: Image, _: Allocator, start_row: u32, start_col: u32, fill_value: T, options: FloodFillOptions)" in zig
    assert "pub const FloodFillOptions = struct" in zig and "27 => error.OutOfBounds" in zig
