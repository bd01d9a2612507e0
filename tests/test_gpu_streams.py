"""The device entry points on non-blocking streams and from several host threads.

Every stream-taking call promises to be asynchronous on the stream it is given and, where it waits (canny, the metrics, svd, find_lines,
the fdm status), to wait for that stream only.  The suite's other tests all run on torch's default stream, the legacy NULL stream, which is
implicitly ordered with every other stream: work the library leaves on the NULL stream and calls that wait for the whole device are
invisible there.  Every kernel here is deterministic (integer atomics, fixed-order f64 partial sums, per-block reductions finished on the
host), so "the same call on another stream or thread gives the same bits" is a strong oracle that covers every op at once.

* test_same_bits_on_non_blocking_stream: each op of OPS on a `torch.cuda.Stream()` (non-blocking) equals its default-stream run bit for bit,
  host scalars and zb_last_kernel() included, and the kernel is the specialised one the op is meant to reach.
* test_no_op_waits_for_other_streams: the whole table, cold (first-use tables, plans and LUTs included), in a fresh subprocess with eager
  module loading, on a non-blocking stream while one single-CTA sleep kernel occupies the NULL stream.  After every call the NULL stream
  must still be busy; afterwards the cold results equal the default-stream ones and the first-use paths match the CPU oracle.
* test_threads_each_with_its_own_stream: four host threads (ctypes releases the GIL, so the library calls overlap), each with its own
  stream, seed and objects, run the table once; every thread's results equal its serial default-stream results.
* test_resize_plan_eviction: more distinct plane resizes than the plan cache holds, then the first again, all against the oracle.

Run as a script (`python tests/test_gpu_streams.py --cold BLOCKER_MS`) the file performs the cold run of the second test and prints a JSON
report; the test starts it that way.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import threading
import time
import zlib
from dataclasses import dataclass
from pathlib import Path
from typing import Callable, Optional

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if __name__ == "__main__":   # the cold run: the same imports the suite gets from tests/conftest.py
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "tests"))

import hough_oracle  # noqa: E402
import oracle_lib as zo  # noqa: E402

pytestmark = pytest.mark.gpu


# ---- inputs ---------------------------------------------------------------------------------------------------------------------

def _u8(rng, shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)


def _f32(rng, shape):
    return rng.random(shape, dtype=np.float32)


def _taps(rng, n):
    k = (rng.random(n) + 0.05).astype(np.float32)
    return (k / k.sum()).astype(np.float32)


def _binary(rng, shape):
    return np.where(rng.random(shape) < 0.3, 255, 0).astype(np.uint8)


def _edges(rng):
    img = np.where(rng.random((150, 170)) < 0.01, rng.integers(1, 256, (150, 170)), 0).astype(np.uint8)
    img[60, 10:150] = 255                                             # a horizontal line
    idx = np.arange(20, 130)
    img[idx, idx + 15] = 200                                          # and a diagonal one
    return img


class _Affine:
    """The transform argument of Image.warp: an affine 2x2 matrix + bias."""

    def __init__(self, m):
        self.m = np.asarray(m, np.float32)

    def as_f32(self):
        return 1, self.m


AFFINE = [0.9, -0.2, 0.25, 1.1, 1.5, -2.0]
HOUGH_SIZE, HOUGH_BOX = 128, (5, 7, 133, 135)


# ---- the op table ---------------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class Op:
    name: str
    build: Callable            # rng -> dict of host inputs: arrays under "img*" become device Images, under "mat*" / "acc" tensors
    run: Callable              # (zb, device inputs) -> dict of outputs (Images, tensors, host values); "_*" entries are kept alive only
    kernel: tuple = ()         # the zb_last_kernel() names the call may report (empty: the op names no kernel of its own)
    knobs: tuple = ()          # process-wide switches set around the call: never inside the threaded test
    oracle: Optional[Callable] = None   # (host inputs, fetched outputs) -> asserts against the CPU oracle (the cold run's first-use paths)


def _sep(border="MIRROR"):
    def run(zb, d):
        return {"out": d["img"].convolve_separable(d["kx"], d["ky"], zb.BorderMode[border])}
    return run


def _tile_u8(zb, d):
    v = d["img"].view(zb.Rectangle(3, 0, 299, 100))                   # 12-byte offset: not TMA-aligned, so the shared-memory tile kernel
    return {"out": v.convolve_separable(d["kx"], d["ky"], zb.BorderMode.WRAP)}


def _resize(shape, method):
    def run(zb, d):
        out = zb.Image.init(shape[0], shape[1], d["img"].pixfmt)
        return {"out": d["img"].resize(out, zb.Interpolation[method.upper()])}

    def oracle(h, o):
        assert np.array_equal(o["out"], zo.resize(h["img"], shape, method))
    return run, oracle


def _warp_lanczos(zb, d):
    out = zb.Image.init(85, 97, d["img"].pixfmt)
    return {"out": d["img"].warp(out, _Affine(AFFINE), zb.Interpolation.LANCZOS)}


def _warp_oracle(h, o):
    assert np.array_equal(o["out"], zo.warp(h["img"], np.zeros((85, 97, 3), np.uint8), "affine", AFFINE, "lanczos"))


def _extract(zb, d):
    out = zb.Image.init(50, 64, d["img"].pixfmt)
    return {"out": d["img"].extract(out, (5.0, 4.0, 85.0, 70.0), 0.3, zb.Interpolation.BILINEAR, zb.BorderMode.ZERO)}


def _insert(zb, d):
    return {"out": d["img"].insert(d["img_src"], (10.0, 12.0, 70.0, 60.0), 0.4, zb.Interpolation.BICUBIC)}


def _motion_linear(zb, d):
    from zignal_b200.compose import motion_blur_linear
    return {"out": motion_blur_linear(d["img"], zb.Image.init_like(d["img"]), 0.7, 5)}


def _motion_radial(spin):
    def run(zb, d):
        from zignal_b200.compose import motion_blur_radial
        return {"out": motion_blur_radial(d["img"], zb.Image.init_like(d["img"]), 0.4, 0.6, 0.5, spin=spin)}
    return run


def _morph(op):
    def run(zb, d):
        return {"out": getattr(d["img"], op)(d["kernel"], 2)}
    return run


def _hough(zb, d):
    h = zb.HoughTransform(HOUGH_SIZE)                                  # a new object: its tables are uploaded by this compute
    h.compute(d["img"], zb.Rectangle(*HOUGH_BOX), d["acc"])
    lines = h.find_lines(d["acc"], 60, 4.0, 3.0)
    return {"acc": d["acc"], "lines": [(l.angle, l.radius, l.score) + l.p1 + l.p2 for l in lines], "_hough": h}


def _hough_oracle(h, o):
    want = hough_oracle.compute(HOUGH_SIZE, h["img"], HOUGH_BOX, np.zeros((HOUGH_SIZE, HOUGH_SIZE), np.uint32))
    assert np.array_equal(o["acc"].view(np.uint32), want)
    assert o["lines"] == hough_oracle.find_lines(HOUGH_SIZE, want, 60, 4.0, 3.0) and o["lines"]


def _fdm(zb, d):
    from zignal_b200.fdm import FeatureDistributionMatching
    f = FeatureDistributionMatching(d["img"].pixfmt)                 # a new object: its device state is created by this set_target / update
    f.set_target(d["img_target"])
    f.set_source(d["img"])
    f.update()
    return {"out": d["img"], "status": f.status(), "_fdm": f}


def _fdm_oracle(h, o):
    diff = o["out"].astype(np.int32) - zo.fdm_match(h["img"], h["img_target"]).astype(np.int32)
    assert np.abs(diff).max() <= 1 and np.count_nonzero(diff) <= 2   # exact integer moments vs Welford: rare one-count flips


def _gemm(ta, tb):
    def run(zb, d):
        from zignal_b200 import matrix
        return {"out": matrix.gemm_device(d["mat_a"], d["mat_b"], ta, tb, 0.5, 0.0, None)}
    return run


def _gemm_xtx(zb, d):
    from zignal_b200 import matrix
    return {"out": matrix.gemm_device(d["mat"], d["mat"], True, False, 1.0, 0.0, None)}   # one tensor as both operands: X^T X


def _center(zb, d):
    import torch
    from zignal_b200 import matrix
    x = d["mat"]
    mean, centered = torch.empty(x.shape[1], dtype=x.dtype, device=x.device), torch.empty_like(x)
    matrix.center_columns(x, mean, True, centered)
    return {"mean": mean, "centered": centered}


def _svd(zb, d):
    from zignal_b200 import matrix
    u, s, v, conv = matrix.svd_device(d["mat"], True, True)
    return {"u": u, "s": s, "v": v, "conv": conv}


def _svd_oracle(h, o):
    a = h["mat"].astype(np.float64)
    tol = 1e-5 if h["mat"].dtype == np.float32 else 1e-12
    want = np.linalg.svd(a, compute_uv=False)
    assert o["conv"] == 0 and np.abs(o["s"] - want).max() <= tol * want[0]
    recon = (o["u"].astype(np.float64) * o["s"]) @ o["v"].astype(np.float64).T
    assert np.abs(recon - a).max() <= 10 * tol * want[0]


def _pca_core(zb, d):
    """Pca.fit's device part (covariance path): centring, X^T X / (n - 1) on the tensor cores, the SVD of the covariance."""
    import torch
    from zignal_b200 import matrix
    x = d["mat"]
    n, dim = x.shape
    mean, centered = torch.empty(dim, dtype=x.dtype, device=x.device), torch.empty_like(x)
    matrix.center_columns(x, mean, True, centered)
    cov = matrix.gemm_device(centered, centered, True, False, 1.0 / (n - 1), 0.0, None)
    u, s, _, conv = matrix.svd_device(cov, True, False)
    return {"mean": mean, "cov": cov, "u": u, "s": s, "conv": conv}


def _pca_oracle(h, o):
    x = h["mat"].astype(np.float64)
    xc = x - x.mean(0)
    cov = xc.T @ xc / (x.shape[0] - 1)
    assert np.abs(o["mean"] - x.mean(0)).max() <= 1e-6 * np.abs(x).max()
    assert np.abs(o["cov"] - cov).max() <= 2e-6 * np.abs(cov).max()
    want = np.linalg.svd(o["cov"].astype(np.float64), compute_uv=False)
    assert o["conv"] == 0 and np.abs(o["s"] - want).max() <= 1e-5 * want[0]


R_PLANE, R_UNIFORM, R_4TO1, R_LANCZOS = _resize((77, 123), "bilinear"), _resize((32, 33), "bicubic"), _resize((16, 256), "bicubic"), \
    _resize((61, 157), "lanczos")
RGBA8_SEP = ("fused_sep_rgba8_dp", "fused_sep_rgba8_f", "fused_sep_rgba8")

# The table runs in this order; in the cold run the generic Lanczos resize is the first Lanczos call of the process (warp the second).
OPS = [
    Op("conv_sep_rgbaf32", lambda r: {"img": _f32(r, (96, 256, 4)), "kx": _taps(r, 7), "ky": _taps(r, 9)}, _sep(), ("fused_sep_rgbaf32",)),
    Op("conv_sep_rgbaf32_exact", lambda r: {"img": _f32(r, (96, 256, 4)), "kx": _taps(r, 7), "ky": _taps(r, 7)}, _sep("REPLICATE"),
       ("fused_sep_rgbaf32_exact",), knobs=(("zb_set_exact_f32", 1),)),
    Op("conv_sep_rgba8", lambda r: {"img": _u8(r, (96, 256, 4)), "kx": _taps(r, 9), "ky": _taps(r, 5)}, _sep(), RGBA8_SEP),
    Op("conv_sep_tile_u8", lambda r: {"img": _u8(r, (100, 304, 4)), "kx": _taps(r, 6), "ky": _taps(r, 15)}, _tile_u8,
       ("sep_tile_u8", "sep_tile_u8_dp")),
    Op("conv_sep_generic_u8", lambda r: {"img": _u8(r, (96, 200, 4)), "kx": (r.standard_normal(5) * 3000).astype(np.float32),
                                         "ky": (r.standard_normal(5) * 3000).astype(np.float32)}, _sep(), ("sep_generic_u8",)),
    Op("conv_sep_generic_f32", lambda r: {"img": _f32(r, (64, 100, 4)), "kx": np.array([0.25, 1e-12, 0.5, 0.0, 0.25], np.float32),
                                          "ky": _taps(r, 3)}, _sep(), ("sep_generic_f32",)),
    Op("convolve_dense_u8", lambda r: {"img": _u8(r, (100, 160, 4)), "k": (r.standard_normal((5, 5)) / 25).astype(np.float32)},
       lambda zb, d: {"out": d["img"].convolve(d["k"], zb.BorderMode.REPLICATE)}, ("conv2d_tile_u8",)),
    Op("convolve_dense_f32", lambda r: {"img": _f32(r, (90, 130)), "k": (r.standard_normal((3, 3)) / 9).astype(np.float32)},
       lambda zb, d: {"out": d["img"].convolve(d["k"], zb.BorderMode.MIRROR)}, ("conv2d_generic_f32",)),
    Op("gaussian_blur_rgba8", lambda r: {"img": _u8(r, (96, 256, 4))}, lambda zb, d: {"out": d["img"].gaussian_blur(1.5)}, RGBA8_SEP),
    Op("gaussian_blur_rgbaf32", lambda r: {"img": _f32(r, (96, 256, 4))}, lambda zb, d: {"out": d["img"].gaussian_blur(2.0)},
       ("fused_sep_rgbaf32",)),
    Op("box_blur_fused", lambda r: {"img": _u8(r, (150, 200))}, lambda zb, d: {"out": d["img"].box_blur(3)}, ("box_fused_blur",)),
    Op("sharpen_fused", lambda r: {"img": _u8(r, (100, 120, 4))}, lambda zb, d: {"out": d["img"].sharpen(2)}, ("box_fused_sharpen",)),
    Op("box_blur_sat", lambda r: {"img": _f32(r, (150, 200))}, lambda zb, d: {"out": d["img"].box_blur(4)}, ("sat_box_blur",)),
    Op("sharpen_sat", lambda r: {"img": _u8(r, (100, 120, 3))}, lambda zb, d: {"out": d["img"].sharpen(2)}, ("sat_sharpen",)),
    Op("resize_plane", lambda r: {"img": _u8(r, (100, 150, 3))}, R_PLANE[0], ("resize_plane_u8",), oracle=R_PLANE[1]),
    Op("resize_uniform_cubic", lambda r: {"img": _u8(r, (96, 99, 4))}, R_UNIFORM[0], ("resize_cubic_uniform_u8",), oracle=R_UNIFORM[1]),
    Op("resize_4to1", lambda r: {"img": _u8(r, (64, 1024, 3))}, R_4TO1[0], ("resize_cubic_r4_u8",), oracle=R_4TO1[1]),
    Op("resize_generic_lanczos", lambda r: {"img": _f32(r, (90, 110))}, R_LANCZOS[0], ("resize_generic",), oracle=R_LANCZOS[1]),
    Op("warp_lanczos", lambda r: {"img": _u8(r, (80, 100, 3))}, _warp_lanczos, ("warp_gather",), oracle=_warp_oracle),
    Op("rotate_tile", lambda r: {"img": _u8(r, (120, 160, 4))}, lambda zb, d: {"out": d["img"].rotate(0.6)}, ("rotate_tile_rgba8",)),
    Op("rotate_gather", lambda r: {"img": _u8(r, (120, 160))},
       lambda zb, d: {"out": d["img"].rotate(0.6, zb.Interpolation.BICUBIC, zb.BorderMode.MIRROR)}, ("rotate_gather",)),
    Op("rotate_orthogonal", lambda r: {"img": _u8(r, (90, 130, 3))}, lambda zb, d: {"out": d["img"].rotate(float(np.float32(np.pi / 2)))},
       ("rotate_orthogonal",)),
    Op("extract", lambda r: {"img": _u8(r, (100, 120, 4))}, _extract, ("extract_gather",)),
    Op("insert", lambda r: {"img": _u8(r, (100, 120, 4)), "img_src": _u8(r, (40, 50, 4))}, _insert, ("insert_gather",)),
    Op("motion_blur_linear", lambda r: {"img": _u8(r, (90, 120, 3))}, _motion_linear, ("motion_line",)),
    Op("motion_blur_zoom", lambda r: {"img": _u8(r, (90, 120, 4))}, _motion_radial(False), ("motion_zoom",)),
    Op("motion_blur_spin", lambda r: {"img": _f32(r, (90, 120))}, _motion_radial(True), ("motion_spin",)),
    Op("sobel", lambda r: {"img": _u8(r, (150, 300))}, lambda zb, d: {"out": d["img"].sobel()}, ("sobel_tile_u8",)),
    Op("canny", lambda r: {"img": _u8(r, (120, 160))}, lambda zb, d: {"out": d["img"].canny(1.0, 20.0, 60.0)}, ("canny",)),
    Op("shen_castan", lambda r: {"img": _u8(r, (120, 160))}, lambda zb, d: {"out": d["img"].shen_castan()}, ("shen_castan",)),
    Op("median_blur", lambda r: {"img": _u8(r, (90, 110, 3))}, lambda zb, d: {"out": d["img"].median_blur(2)}, ("order_statistic",)),
    Op("alpha_trimmed_mean_blur", lambda r: {"img": _u8(r, (90, 110))}, lambda zb, d: {"out": d["img"].alpha_trimmed_mean_blur(4, 0.2)},
       ("order_statistic",)),
    Op("psnr", lambda r: {"img": _u8(r, (100, 130, 3)), "img_b": _u8(r, (100, 130, 3))}, lambda zb, d: {"v": d["img"].psnr(d["img_b"])},
       ("diff_sums",)),
    Op("ssim", lambda r: {"img": _f32(r, (100, 130)), "img_b": _f32(r, (100, 130))}, lambda zb, d: {"v": d["img"].ssim(d["img_b"])},
       ("ssim",)),
    Op("mean_pixel_error", lambda r: {"img": _f32(r, (100, 130, 4)), "img_b": _f32(r, (100, 130, 4))},
       lambda zb, d: {"v": d["img"].mean_pixel_error(d["img_b"])}, ("diff_sums",)),
    Op("convert", lambda r: {"img": _u8(r, (100, 130, 3))}, lambda zb, d: {"out": d["img"].convert(zb.PixFmt.RGBAF32)}, ("convert",)),
    Op("histogram", lambda r: {"img": _u8(r, (100, 130, 4))}, lambda zb, d: {"v": d["img"].histogram()}, ("histogram",)),
    Op("equalize", lambda r: {"img": (_u8(r, (100, 130, 3)) // 3 + 40).astype(np.uint8)}, lambda zb, d: {"out": d["img"].equalize()},
       ("equalize",)),
    Op("autocontrast", lambda r: {"img": (_u8(r, (100, 130, 4)) // 2 + 30).astype(np.uint8)},
       lambda zb, d: {"out": d["img"].autocontrast(0.02)}, ("autocontrast",)),
    Op("threshold_otsu", lambda r: {"img": _u8(r, (120, 150))}, lambda zb, d: dict(zip(("out", "t"), d["img"].threshold_otsu())),
       ("threshold_otsu",)),
    Op("threshold_adaptive_mean", lambda r: {"img": _u8(r, (120, 152))},   # 4-byte rows: the fused path
       lambda zb, d: {"out": d["img"].threshold_adaptive_mean(5, 3.0)}, ("box_fused_threshold",)),
    Op("dilate_binary", lambda r: {"img": _binary(r, (120, 150)), "kernel": np.ones((3, 3), np.uint8)}, _morph("dilate_binary"),
       ("morph_binary",)),
    Op("erode_binary", lambda r: {"img": _binary(r, (120, 150)), "kernel": np.ones((5, 3), np.uint8)}, _morph("erode_binary"),
       ("morph_binary",)),
    Op("open_binary", lambda r: {"img": _binary(r, (120, 150)), "kernel": np.ones((3, 3), np.uint8)}, _morph("open_binary"),
       ("morph_binary",)),
    Op("close_binary", lambda r: {"img": _binary(r, (120, 150)), "kernel": np.ones((3, 5), np.uint8)}, _morph("close_binary"),
       ("morph_binary",)),
    Op("hough", lambda r: {"img": _edges(r), "acc": np.zeros((HOUGH_SIZE, HOUGH_SIZE), np.int32)}, _hough, ("hough_vote",),
       oracle=_hough_oracle),
    Op("fdm", lambda r: {"img": _u8(r, (120, 150, 3)), "img_target": (_u8(r, (120, 150, 3)) // 2 + 40).astype(np.uint8)}, _fdm,
       ("fdm_map",), oracle=_fdm_oracle),
    Op("gemm_f32", lambda r: {"mat_a": r.standard_normal((70, 300)).astype(np.float32), "mat_b": r.standard_normal((300, 65)).astype(np.float32)},
       _gemm(False, False), ("gemm_f32_acc64",)),
    Op("gemm_f64", lambda r: {"mat_a": r.standard_normal((70, 300)), "mat_b": r.standard_normal((65, 300))}, _gemm(False, True),
       ("gemm_f64",)),
    Op("gemm_xtx", lambda r: {"mat": r.standard_normal((4096, 128)).astype(np.float32)}, _gemm_xtx, ("gemm_xtx_tf32x3_wgmma",)),
    Op("center_columns", lambda r: {"mat": r.standard_normal((500, 12))}, _center),
    Op("svd_device_f32", lambda r: {"mat": r.standard_normal((96, 64)).astype(np.float32)}, _svd, ("jacobi_svd_cluster",), oracle=_svd_oracle),
    Op("svd_device_f64", lambda r: {"mat": r.standard_normal((60, 24))}, _svd, ("jacobi_svd_onesided",), oracle=_svd_oracle),
    Op("pca_fit_core", lambda r: {"mat": (r.standard_normal((4096, 128)) @ r.standard_normal((128, 128))).astype(np.float32)}, _pca_core,
       ("jacobi_svd_cluster",), oracle=_pca_oracle),
]
OPS_BY_NAME = {op.name: op for op in OPS}
assert len(OPS_BY_NAME) == len(OPS)


# ---- running, fetching and comparing --------------------------------------------------------------------------------------------

def _seed(name: str, base: int = 0) -> int:
    return zlib.crc32(name.encode()) ^ base


def _host_inputs(op: Op, base: int = 0) -> dict:
    return op.build(np.random.default_rng(_seed(op.name, base)))


def _prepare(zb, host: dict) -> dict:
    """Device copies of the host inputs, on the current stream."""
    import torch
    dev = {}
    for k, v in host.items():
        if isinstance(v, np.ndarray) and (k.startswith("mat") or k == "acc"):
            dev[k] = torch.from_numpy(v).cuda()
        elif isinstance(v, np.ndarray) and k.startswith("img"):
            dev[k] = zb.Image.from_numpy(v)
        else:
            dev[k] = v
    return dev


def _call(zb, op: Op, dev: dict):
    """One call of the op -> (outputs, zb_last_kernel()).  The knobs are process-wide: set around the call, then restored."""
    L = zb.lib()
    for fn, value in op.knobs:
        getattr(L, fn)(value)
    try:
        out = op.run(zb, dev)
        return out, L.zb_last_kernel().decode()
    finally:
        for fn, _ in op.knobs:
            getattr(L, fn)(0)


def _fetch(out: dict) -> dict:
    """Host copies of the outputs (on the current stream, which the device copies wait for)."""
    import torch
    res = {}
    for k, v in out.items():
        if k.startswith("_"):
            continue
        if isinstance(v, torch.Tensor):
            res[k] = v.cpu().numpy()
        elif hasattr(v, "to_numpy"):
            res[k] = v.to_numpy()
        else:
            res[k] = v
    return res


def _release(out: dict) -> None:
    for k, v in out.items():
        if k.startswith("_"):
            v.deinit()


def _run(zb, op: Op, host: dict):
    """Prepare, call, fetch on the current stream -> (host outputs, kernel name)."""
    out, kernel = _call(zb, op, _prepare(zb, host))
    res = _fetch(out)
    _release(out)
    return res, kernel


def _same(a, b) -> bool:
    """Bit equality of fetched outputs (arrays: dtype, shape and bytes; floats: bytes, so inf / nan compare too)."""
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return (isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape
                and a.tobytes() == b.tobytes())
    if isinstance(a, float) or isinstance(b, float):
        return np.float64(a).tobytes() == np.float64(b).tobytes()
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return type(a) is type(b) and a == b


def _diff(want: dict, got: dict) -> list:
    return sorted(k for k in set(want) | set(got) if k not in want or k not in got or not _same(want[k], got[k]))


# ---- a. the same bits on a non-blocking stream ----------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    zb.lib().zb_set_exact_f32(0)
    return zb


@pytest.mark.parametrize("name", [op.name for op in OPS])
def test_same_bits_on_non_blocking_stream(zb, name):
    import torch
    op = OPS_BY_NAME[name]
    host = _host_inputs(op)
    want, want_kernel = _run(zb, op, host)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got, got_kernel = _run(zb, op, host)
    assert got_kernel == want_kernel, (want_kernel, got_kernel)
    if op.kernel:
        assert want_kernel in op.kernel, want_kernel
    assert not _diff(want, got), _diff(want, got)


# ---- b. no call waits for other streams -----------------------------------------------------------------------------------------

def _cycles_per_ms(torch) -> float:
    """torch.cuda._sleep spins a single thread for a number of clock cycles: its rate, from an event-timed short sleep."""
    with torch.cuda.stream(torch.cuda.default_stream()):
        torch.cuda._sleep(1000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.cuda._sleep(5_000_000)
        e1.record()
    e1.synchronize()
    return 5_000_000 / max(e0.elapsed_time(e1), 1e-3)


def _block(torch, cycles: int) -> float:
    """One sleep kernel (one CTA) on the legacy NULL stream; returns the host time it was queued at."""
    with torch.cuda.stream(torch.cuda.default_stream()):
        torch.cuda._sleep(cycles)
    return time.perf_counter()


def _warm_torch_allocator(torch) -> None:
    """Let torch's caching allocator hold enough memory on the current stream that the table's output tensors come from its cache:
    a cudaMalloc of torch's own inside the timed window is not what the test is about."""
    big = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    small = [torch.empty(1 << 20, dtype=torch.uint8, device="cuda") for _ in range(128)]
    del big, small


def _cold_main(blocker_ms: float) -> int:
    """The cold run of test_no_op_waits_for_other_streams, in a fresh process: prints a JSON report, exits non-zero on a failure."""
    import ctypes
    import torch
    import zignal_b200 as zb
    zb.lib().zb_set_exact_f32(0)
    # The library's first CUDA runtime call in a process loads its kernels (all of them under eager module loading), and loading a module
    # waits for the device.  That start-up cost is paid here, before the blocker; the first-use tables, plans and LUTs stay cold.
    zb._ffi.check(zb.lib().zb_sm_count(ctypes.byref(ctypes.c_int())))
    s = torch.cuda.Stream()
    hosts = [_host_inputs(op) for op in OPS]
    with torch.cuda.stream(s):
        devs = [_prepare(zb, h) for h in hosts]
        _warm_torch_allocator(torch)
    s.synchronize()
    cycles = int(blocker_ms * _cycles_per_ms(torch))
    torch.cuda.synchronize()

    report = {"blocker_ms": blocker_ms, "waited": [], "blocker_too_short": [], "mismatch": [], "oracle": [], "kernel": []}
    outs = []
    with torch.cuda.stream(s):
        started = _block(torch, cycles)
        for op, dev in zip(OPS, devs):
            t0 = time.perf_counter()
            out, kernel = _call(zb, op, dev)
            t1 = time.perf_counter()
            if torch.cuda.default_stream().query():   # the blocker is done: this call waited for it, or the blocker was too short
                call_ms, since_ms = 1e3 * (t1 - t0), 1e3 * (t1 - started)
                entry = {"op": op.name, "call_ms": round(call_ms, 1), "since_blocker_ms": round(since_ms, 1)}
                report["waited" if call_ms > 0.25 * blocker_ms else "blocker_too_short"].append(entry)
                started = _block(torch, cycles)       # a new blocker, so the ops after this one are still checked
            outs.append((out, kernel))
        s.synchronize()
        report["blocker_alive_at_end"] = not torch.cuda.default_stream().query()
        cold = [(_fetch(out), kernel) for out, kernel in outs]
    torch.cuda.synchronize()
    for out, _ in outs:                                   # destroy functions synchronise the device: only now
        _release(out)

    for op, host, (got, got_kernel) in zip(OPS, hosts, cold):
        want, want_kernel = _run(zb, op, host)            # the same op, warm, on the default stream
        if _diff(want, got):
            report["mismatch"].append({"op": op.name, "outputs": _diff(want, got)})
        if got_kernel != want_kernel or (op.kernel and got_kernel not in op.kernel):
            report["kernel"].append({"op": op.name, "cold": got_kernel, "default_stream": want_kernel})
        if op.oracle is not None:
            try:
                op.oracle(host, got)
            except AssertionError as e:
                report["oracle"].append({"op": op.name, "error": repr(e)[:300]})
    print(json.dumps(report))
    ok = not (report["waited"] or report["blocker_too_short"] or report["mismatch"] or report["oracle"] or report["kernel"])
    return 0 if ok and report["blocker_alive_at_end"] else 1


def test_no_op_waits_for_other_streams(zb):
    """The table cold, on a non-blocking stream, while a sleep kernel holds the legacy NULL stream (see _cold_main).  The blocker is sized
    from this process's warm run of the table: ten times that, at least one second, at most four."""
    import torch
    hosts = [_host_inputs(op) for op in OPS]
    for op, host in zip(OPS, hosts):                       # warm-up, then the timed pass
        _run(zb, op, host)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for op, host in zip(OPS, hosts):
        _run(zb, op, host)
    torch.cuda.synchronize()
    blocker_ms = min(max(10 * 1e3 * (time.perf_counter() - t0), 1000.0), 4000.0)
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER")    # lazy loading may synchronise the context on a kernel's first launch
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, str(Path(__file__).resolve()), "--cold", f"{blocker_ms:.0f}"], env=env, cwd=str(ROOT),
                       capture_output=True, text=True, timeout=900)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert lines, f"no report (exit {r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    report = json.loads(lines[-1])
    assert not report["waited"], f"calls that waited for the NULL stream: {report['waited']}"
    assert not report["blocker_too_short"], report
    assert report["blocker_alive_at_end"], report
    assert not report["mismatch"] and not report["kernel"] and not report["oracle"], report
    assert r.returncode == 0, r.stderr[-3000:]


# ---- c. several host threads ----------------------------------------------------------------------------------------------------

def test_threads_each_with_its_own_stream(zb):
    """Four threads, each with its own stream, seed, inputs and Hough / fdm objects, run the table once (no repeat loops: a contract
    check, not a race hunt).  Ops that need a process-wide knob are left out: a knob set by one thread would change another's call."""
    import torch
    ops = [op for op in OPS if not op.knobs]
    seeds = (101, 202, 303, 404)
    hosts = {seed: [_host_inputs(op, seed) for op in ops] for seed in seeds}
    serial = {seed: [_run(zb, op, h) for op, h in zip(ops, hosts[seed])] for seed in seeds}
    torch.cuda.synchronize()
    results, errors = {}, []
    start = threading.Barrier(len(seeds))

    def work(seed):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                devs = [_prepare(zb, h) for h in hosts[seed]]
                s.synchronize()
                start.wait()
                outs = [_call(zb, op, dev) for op, dev in zip(ops, devs)]
                s.synchronize()
                results[seed] = [(_fetch(out), kernel) for out, kernel in outs]
            results[seed, "objects"] = [out for out, _ in outs]
        except BaseException as e:   # noqa: B902 -- reported by the main thread
            errors.append((seed, repr(e)))
            start.abort()

    threads = [threading.Thread(target=work, args=(seed,)) for seed in seeds]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for seed in seeds:
        for out in results.get((seed, "objects"), []):
            _release(out)
    assert not errors, errors
    bad = []
    for seed in seeds:
        for op, (want, want_kernel), (got, got_kernel) in zip(ops, serial[seed], results[seed]):
            if _diff(want, got) or got_kernel != want_kernel or (op.kernel and got_kernel not in op.kernel):
                bad.append((seed, op.name, _diff(want, got), want_kernel, got_kernel))
    assert not bad, bad


# ---- d. resize plan eviction ----------------------------------------------------------------------------------------------------

def test_resize_plan_eviction(zb):
    """The Rgb / Rgba u8 resizers cache up to 32 plans (tap tables on the device).  40 distinct (shape, method) resizes evict the oldest
    ones; the first resize, run again, builds its plan anew.  Every result equals the oracle's."""
    methods = ["nearest", "bilinear", "bicubic", "catmull_rom", "mitchell", "lanczos"]
    rng = np.random.default_rng(40)
    cases = [((23 + i, 31 + 2 * i, 3 + i % 2), (11 + (7 * i) % 29, 17 + (5 * i) % 31), methods[i % len(methods)]) for i in range(40)]
    assert len({(src[:2], dst, m) for src, dst, m in cases}) == 40 and all(src[:2] != dst for src, dst, _ in cases)   # 40 plans
    for src_shape, dst_shape, method in cases + cases[:1]:
        img = _u8(rng, src_shape)
        dev = zb.Image.from_numpy(img)
        got = dev.resize(zb.Image.init(dst_shape[0], dst_shape[1], dev.pixfmt), zb.Interpolation[method.upper()]).to_numpy()
        assert np.array_equal(got, zo.resize(img, dst_shape, method)), (src_shape, dst_shape, method)


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--cold":
        sys.exit("usage: test_gpu_streams.py --cold BLOCKER_MS")
    sys.exit(_cold_main(float(sys.argv[2])))
