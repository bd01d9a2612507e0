"""CPU checks of colour quantization and dithering: the reference's own tests (sixel, GIF and quantize tests) as known answers on the oracle
(oracle/zo_quantize.cpp), an independent pure-Python restatement that pins the oracle (std.sort.heap and median cut, a brute-force argmin
LUT, per-pixel diffusion loops) over every mode, all fixed palettes, palettes of 1, 2, 16 and 256 entries and palettes with duplicates,
targeted cases (an unstable-sort tie that changes the palette, per-contribution clamps against sum-then-clamp, 1 x N, N x 1 and 2 x 2
images, Atkinson on one row), the golden fixtures, the new status name and the argument errors the library decides before any device
work."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

import quantize_oracle as zo
from golden_quantize import CASES, DITHER_MODES, all_bins_shuffled, palette, random_palette, run_chain, smooth_rgb
from gpu_utils import sha

GOLDEN = Path(__file__).resolve().parent / "golden" / "golden_quantize.json"

# ---- the independent restatement --------------------------------------------------------------------------------------------------------


def py_heap_sort(items, less):
    """std.sort.heap: heapify with siftDown from len/2 - 1 down to 0, then swap the root to the end and sift down."""
    items = list(items)

    def sift(cur, end):
        while True:
            child = 2 * cur + 1
            if child >= end:
                return
            if child + 1 < end and less(items[child], items[child + 1]):
                child += 1
            if less(items[child], items[cur]):
                return
            items[child], items[cur] = items[cur], items[child]
            cur = child

    for i in reversed(range(len(items) // 2)):
        sift(i, len(items))
    for end in reversed(range(1, len(items))):
        items[0], items[end] = items[end], items[0]
        sift(0, end)
    return items


def py_color_list(img):
    """(r8, g8, b8, count) per touched 5-bit key, in first-touch raster order."""
    keys = ((img[..., 0].astype(np.int64) >> 3) << 10 | (img[..., 1].astype(np.int64) >> 3) << 5 | (img[..., 2].astype(np.int64) >> 3)).ravel()
    uniq, first, counts = np.unique(keys, return_index=True, return_counts=True)
    order = np.argsort(first)
    out = []
    for k, n in zip(uniq[order], counts[order]):
        r5, g5, b5 = (int(k) >> 10) & 31, (int(k) >> 5) & 31, int(k) & 31
        out.append(((r5 << 3) | (r5 >> 2), (g5 << 3) | (g5 >> 2), (b5 << 3) | (b5 >> 2), int(n)))
    return out


def py_median_cut(img, max_colors, cap=256, stable=False):
    colors = py_color_list(img)
    size = min(len(colors), max_colors, cap)
    if size == 0:
        return None
    if len(colors) == 1:
        return np.array([colors[0][:3]], np.uint8)

    def box(lst):
        if not lst:
            return {"c": lst, "min": [255] * 3, "max": [0] * 3, "pop": 0}
        return {"c": lst, "min": [min(c[k] for c in lst) for k in range(3)], "max": [max(c[k] for c in lst) for k in range(3)],
                "pop": sum(c[3] for c in lst)}

    boxes = [box(colors)]
    while len(boxes) < size:
        best, best_score = None, 0
        for i, b in enumerate(boxes):
            if len(b["c"]) <= 1 or all(b["max"][k] <= b["min"][k] for k in range(3)):
                continue
            vol = 1
            for k in range(3):
                vol *= b["max"][k] - b["min"][k] + 1
            if vol * b["pop"] > best_score:
                best, best_score = i, vol * b["pop"]
        if best is None:
            break
        b = boxes.pop(best)
        rng = [b["max"][k] - b["min"][k] for k in range(3)]
        dim = 1 if rng[1] >= rng[0] and rng[1] >= rng[2] else (0 if rng[0] >= rng[2] else 2)
        cs = sorted(b["c"], key=lambda c: c[dim]) if stable else py_heap_sort(b["c"], lambda x, y: x[dim] < y[dim])
        half = sum(c[3] for c in cs) // 2
        acc, cut = 0, 0
        for i, c in enumerate(cs):
            acc += c[3]
            if acc >= half:
                cut = max(1, min(i + 1, len(cs) - 1))
                break
        boxes += [box(cs[:cut]), box(cs[cut:])]
    pal = []
    for b in boxes[:min(len(boxes), cap)]:
        w = sum(c[3] for c in b["c"])
        pal.append([sum(c[k] * c[3] for c in b["c"]) // w for k in range(3)])
    return np.array(pal, np.uint8).reshape(-1, 3)


def py_lut(pal):
    pal = np.asarray(pal, np.int64).reshape(-1, 3)
    v = np.arange(32)
    v8 = (v << 3) | (v >> 2)
    rgb = np.stack(np.meshgrid(v8, v8, v8, indexing="ij"), axis=-1).reshape(-1, 3)
    d = ((rgb[:, None, :] - pal[None, :, :]) ** 2).sum(axis=2)
    return np.argmin(d, axis=1).astype(np.uint8)                    # first minimum: the lowest index on ties


def _padded(pal):
    out = np.zeros((256, 3), np.uint8)
    out[:len(pal)] = pal
    return out


def _key(px):
    return (int(px[0]) >> 3) << 10 | (int(px[1]) >> 3) << 5 | (int(px[2]) >> 3)


def py_dither(img, pal, lut, mode, sum_then_clamp=False):
    img = img.astype(np.int64)
    pal = _padded(pal).astype(np.int64)
    rows, cols = img.shape[:2]
    if mode == zo.ORDERED:
        bayer = np.array([[0, 32, 8, 40, 2, 34, 10, 42], [48, 16, 56, 24, 50, 18, 58, 26], [12, 44, 4, 36, 14, 46, 6, 38],
                          [60, 28, 52, 20, 62, 30, 54, 22], [3, 35, 11, 43, 1, 33, 9, 41], [51, 19, 59, 27, 49, 17, 57, 25],
                          [15, 47, 7, 39, 13, 45, 5, 37], [63, 31, 55, 23, 61, 29, 53, 21]])
        off = (bayer[np.arange(rows)[:, None] & 7, np.arange(cols)[None, :] & 7] - 32) >> 1
        q = np.clip(img + off[..., None], 0, 255) >> 3
        return pal[lut[(q[..., 0] << 10) | (q[..., 1] << 5) | q[..., 2]]].astype(np.uint8)
    if mode not in (zo.FLOYD_STEINBERG, zo.ATKINSON):
        return img.astype(np.uint8)
    dists = ([(1, 0, 7), (-1, 1, 3), (0, 1, 5), (1, 1, 1)], 4) if mode == zo.FLOYD_STEINBERG else \
        ([(1, 0, 1), (2, 0, 1), (-1, 1, 1), (0, 1, 1), (1, 1, 1), (0, 2, 1)], 3)
    pending = np.zeros_like(img)
    for r in range(rows):
        for c in range(cols):
            cur = np.clip(img[r, c] + pending[r, c], 0, 255) if sum_then_clamp else img[r, c].copy()
            q = pal[lut[_key(cur)]]
            img[r, c] = q
            err = cur - q
            for dx, dy, w in dists[0]:
                nr, nc = r + dy, c + dx
                if 0 <= nr < rows and 0 <= nc < cols:
                    contrib = np.trunc(err * w / (1 << dists[1])).astype(np.int64)
                    if sum_then_clamp:
                        pending[nr, nc] += contrib
                    else:
                        img[nr, nc] = np.clip(img[nr, nc] + contrib, 0, 255)
    return img.astype(np.uint8)


# ---- the reference's tests as known answers ---------------------------------------------------------------------------------------------

EIGHT = np.array([[0, 0, 0], [255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [255, 0, 255], [0, 255, 255], [255, 255, 255]], np.uint8)


def test_reference_sixel_adaptive_four_colours():
    img = EIGHT[np.arange(16) % 8].reshape(4, 4, 3)
    pal = zo.build_palette(img, zo.ADAPTIVE, 4)
    assert 1 <= len(pal) <= 4
    assert np.array_equal(pal, py_median_cut(img, 4))


def test_reference_fixed_6x7x6_black_white_red():
    pal = zo.build_palette(None, zo.FIXED_6X7X6)
    assert len(pal) == 252
    lut = zo.color_lut(pal)
    idx = zo.palette_lookup(np.array([[[0, 0, 0], [255, 255, 255], [255, 0, 0]]], np.uint8), lut)
    assert [tuple(int(x) for x in pal[i]) for i in idx[0]] == [(0, 0, 0), (255, 255, 255), (255, 0, 0)]


def test_reference_single_colour():
    img = np.full((4, 4, 3), (10, 20, 30), np.uint8)                # one entry: the colour of the 5-bit bin
    assert zo.median_cut(img, 16).tolist() == [[8, 16, 24]]
    assert zo.build_palette(img, zo.ADAPTIVE, 256).tolist() == [[8, 16, 24]]


def test_reference_gif_gradient_and_floyd_steinberg():
    rr, cc = np.mgrid[0:16, 0:16]
    grad = np.stack([rr * 16, cc * 16, (rr + cc) * 8], axis=2).astype(np.uint8)
    pal = zo.median_cut(grad, 256)
    assert 1 <= len(pal) <= 256 and np.array_equal(pal, py_median_cut(grad, 256))
    img = EIGHT[(np.arange(64) * 5) % 8].reshape(8, 8, 3)
    pal8 = zo.median_cut(img, 8)
    assert len(pal8) == 8
    lut = zo.color_lut(pal8)
    out = zo.dither(img.copy(), pal8, lut, zo.FLOYD_STEINBERG)
    assert np.array_equal(out, img)                                  # every pixel is a palette colour: no error to diffuse
    assert np.array_equal(out, py_dither(img, pal8, lut, zo.FLOYD_STEINBERG))


# ---- the oracle against the restatement -------------------------------------------------------------------------------------------------

def test_heap_sort_matches_restatement():
    rng = np.random.default_rng(0)
    for n in (0, 1, 2, 3, 7, 8, 33, 100):
        a = rng.integers(0, 8, n).astype(np.uint8)
        assert zo.heap_sort_u8(a).tolist() == py_heap_sort(a.tolist(), lambda x, y: x < y) == sorted(a.tolist())


@pytest.mark.parametrize("seed", range(6))
def test_median_cut_matches_restatement(seed):
    rng = np.random.default_rng(seed)
    img = smooth_rgb(13 + seed, 17, seed) if seed % 2 else rng.integers(0, 256, (11, 19, 3), dtype=np.uint8)
    for k in (0, 1, 2, 3, 5, 16, 64, 256):
        for cap in (256, max(k - 1, 0)):
            want = py_median_cut(img, k, cap)
            if want is None:
                with pytest.raises(zo.OracleStatus) as e:
                    zo.median_cut(img, k, cap)
                assert e.value.status == zo.NO_PALETTE_COLORS
            else:
                assert np.array_equal(zo.median_cut(img, k, cap), want), (k, cap)


def test_median_cut_all_bins():
    img = all_bins_shuffled(3)[:64]                                  # 16384 pixels over many bins, in shuffled order
    for k in (2, 9, 40):
        assert np.array_equal(zo.median_cut(img, k), py_median_cut(img, k))


def test_heap_sort_decides_the_palette():
    """Ties in the split dimension: std.sort.heap orders them differently from a stable sort, and that changes which colours share a
    box.  Find such an image among seeded ones and check the oracle follows the heap sort."""
    for seed in range(200):
        rng = np.random.default_rng(seed)
        img = (rng.integers(0, 4, (6, 6, 3)) * 64).astype(np.uint8)
        heap, stable = py_median_cut(img, 5), py_median_cut(img, 5, stable=True)
        if not np.array_equal(heap, stable):
            assert np.array_equal(zo.median_cut(img, 5), heap)
            return
    pytest.fail("no seed separates the heap sort from a stable sort")


PALETTES = ["6x7x6", "vga16", "web216", "random1", "random2", "random16", "random256"]


@pytest.mark.parametrize("kind", PALETTES + ["dup"])
def test_lut_matches_brute_force(kind):
    pal = random_palette(40, 3) if kind == "dup" else palette(kind)
    if kind == "dup":
        pal[20:] = pal[:20]
    assert np.array_equal(zo.color_lut(pal), py_lut(pal))


@pytest.mark.parametrize("mode", DITHER_MODES)
@pytest.mark.parametrize("kind", PALETTES + ["dup"])
def test_dither_matches_restatement(mode, kind):
    pal = random_palette(24, 4) if kind == "dup" else palette(kind)
    if kind == "dup":
        pal[12:] = pal[:12]
    lut = zo.color_lut(pal)
    for k, shape in enumerate(((1, 1), (1, 9), (9, 1), (2, 2), (3, 3), (7, 12), (12, 7))):
        img = smooth_rgb(*shape, k) if k % 2 else np.random.default_rng(k).integers(0, 256, shape + (3,), dtype=np.uint8)
        assert np.array_equal(zo.dither(img.copy(), pal, lut, mode), py_dither(img, pal, lut, mode)), shape


def test_dither_strided_view_matches_contiguous():
    big = smooth_rgb(20, 30, 2)
    pal = palette("vga16")
    lut = zo.color_lut(pal)
    for mode in (zo.FLOYD_STEINBERG, zo.ATKINSON, zo.ORDERED):
        a = big.copy()
        zo.dither(a[3:15, 5:25], pal, lut, mode)
        want = big.copy()
        want[3:15, 5:25] = zo.dither(np.ascontiguousarray(big[3:15, 5:25]), pal, lut, mode)
        assert np.array_equal(a, want)


def test_per_contribution_clamps_matter():
    """Adding the clamped contributions one by one differs from clamping their sum: find seeded near-saturated images where the two
    disagree under a palette far from them, and check the oracle follows the sequence."""
    pal = np.array([[0, 0, 0], [96, 96, 96]], np.uint8)
    lut = zo.color_lut(pal)
    for mode in (zo.FLOYD_STEINBERG, zo.ATKINSON):
        for seed in range(200):
            img = np.random.default_rng(seed).choice(np.array([0, 40, 250, 255], np.uint8), (5, 5, 3))
            seq = py_dither(img, pal, lut, mode)
            if not np.array_equal(seq, py_dither(img, pal, lut, mode, sum_then_clamp=True)):
                assert np.array_equal(zo.dither(img.copy(), pal, lut, mode), seq), mode
                break
        else:
            pytest.fail(f"no seed separates the per-contribution clamps from sum-then-clamp (mode {mode})")


def test_atkinson_one_row_takes_the_checked_branch():
    pal = palette("vga16")
    lut = zo.color_lut(pal)
    for cols in (1, 2, 3, 8, 33):
        img = smooth_rgb(1, cols, cols)
        assert np.array_equal(zo.dither(img.copy(), pal, lut, zo.ATKINSON), py_dither(img, pal, lut, zo.ATKINSON))


def test_lut_index_past_the_palette_reads_zeros():
    """A LUT built for 16 colours used with a 4-colour palette: indices >= 4 read the zero padding."""
    pal16 = palette("vga16")
    lut = zo.color_lut(pal16)
    img = np.full((2, 3, 3), 255, np.uint8)                         # white: index 15
    assert np.array_equal(zo.dither(img.copy(), pal16[:4], lut, zo.ORDERED), np.zeros_like(img))


def test_golden_fixtures():
    gold = json.loads(GOLDEN.read_text())["cases"]
    assert set(gold) == set(CASES)
    for name, (builder, _, _) in CASES.items():
        img = builder()
        pal, lut, idx, out = run_chain(name, img)
        g = gold[name]
        assert (sha(img), sha(pal), sha(lut), sha(idx), sha(out)) == (g["input_sha256"], g["palette_sha256"], g["lut_sha256"],
                                                                       g["indices_sha256"], g["dithered_sha256"]), name


# ---- the library: status name and argument errors (decided before any device work) ------------------------------------------------------

@pytest.fixture(scope="module")
def L():
    from zignal_b200 import _ffi
    if not _ffi.LIB_PATH.exists():
        pytest.skip("libzignal_b200.so not built")
    return _ffi.lib()


def test_status_name(L):
    assert L.zb_status_name(28).decode() == "NoPaletteColors"


def test_argument_errors(L):
    from zignal_b200 import ZbImage
    pal = np.zeros((4, 3), np.uint8)
    p = pal.ctypes.data
    buf = np.zeros(64, np.uint8)
    img = ZbImage(buf.ctypes.data, 4, 4, 4)
    empty = ZbImage(None, 0, 5, 5)
    n = C.c_uint32(0)
    lut = buf.ctypes.data                                            # never dereferenced: every call below fails its checks first
    assert L.zb_color_lut(None, 4, lut, None) == 5
    assert L.zb_color_lut(p, 0, lut, None) == 5
    assert L.zb_color_lut(p, 257, lut, None) == 5
    assert L.zb_color_lut(p, 4, None, None) == 5
    assert L.zb_dither(None, 2, p, 4, lut, 1, None) == 5
    assert L.zb_dither(C.byref(img), 2, p, 4, lut, 5, None) == 5
    assert L.zb_dither(C.byref(img), 2, p, 4, lut, -1, None) == 5
    assert L.zb_dither(C.byref(img), 2, p, 0, lut, 1, None) == 5
    assert L.zb_dither(C.byref(img), 0, p, 4, lut, 1, None) == 3
    assert L.zb_dither(C.byref(img), 3, p, 4, lut, 3, None) == 3
    assert L.zb_dither(C.byref(img), 2, p, 4, lut, 0, None) == 0     # NONE and AUTO do nothing
    assert L.zb_dither(C.byref(img), 2, p, 4, lut, 4, None) == 0
    assert L.zb_palette_lookup(C.byref(img), 2, lut, C.byref(ZbImage(buf.ctypes.data, 4, 5, 5)), None) == 1
    assert L.zb_palette_lookup(C.byref(img), 9, lut, C.byref(img), None) == 3
    assert L.zb_palette_lookup(C.byref(img), 2, None, C.byref(img), None) == 5
    assert L.zb_median_cut(None, 2, 4, p, 4, C.byref(n), None) == 5
    assert L.zb_median_cut(C.byref(img), 9, 4, p, 4, C.byref(n), None) == 3
    assert L.zb_median_cut(C.byref(img), 2, 4, None, 4, C.byref(n), None) == 5
    assert L.zb_median_cut(C.byref(ZbImage(buf.ctypes.data, 65536, 65536, 65536)), 2, 4, p, 4, C.byref(n), None) == 3
    assert L.zb_median_cut(C.byref(empty), 2, 4, p, 4, C.byref(n), None) == 28
    assert L.zb_build_palette(C.byref(img), 2, 7, 4, p, C.byref(n), None) == 5
    out = np.zeros((256, 3), np.uint8)
    for mode, count in ((0, 252), (1, 16), (2, 216)):
        assert L.zb_build_palette(None, 2, mode, 0, out.ctypes.data, C.byref(n), None) == 0
        assert n.value == count and np.array_equal(out[:count], zo.build_palette(None, mode))
    assert L.zb_build_palette(C.byref(empty), 2, 3, 16, out.ctypes.data, C.byref(n), None) == 0   # medianCut fails: 6x7x6
    assert n.value == 252 and np.array_equal(out[:252], zo.build_palette(None, zo.FIXED_6X7X6))
